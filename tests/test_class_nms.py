"""Class-aware NMS in detection: tools/class_nms_oracle.py against torchvision's per-class NMS (the fixture written by
tests/golden/make_class_nms_golden.py), against Soft-NMS run class by class and against a stable argsort; the
refusals of the settings and of the C entries; and -- on the GPU -- the per-class NMS, per-class Soft-NMS and
multi-label top-k kernels against the oracle bit for bit (rows, order and counts), end to end on network outputs,
through GraphedDetect and through evaluate() / evaluate_coco()."""
import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(REPO, 'tools'))
import class_nms_oracle as C  # noqa: E402
import soft_nms_oracle as S  # noqa: E402

gpu = pytest.mark.gpu
IOU = 0.5


def _fixture():
    return np.load(os.path.join(HERE, 'golden', 'class_nms.npz'))


def _case(st, name):
    """(boxes, scores, classes) of a fixture case, regenerated from its seed for the random ones"""
    p = name + '/'
    seed = int(st[p + 'seed'][0])
    if seed < 0:
        return st[p + 'boxes'], st[p + 'scores'], st[p + 'classes']
    b, s, c = C.random_class_candidates(seed, int(st[p + 'n'][0]), int(st[p + 'K'][0]))
    h = hashlib.sha256()
    for x in (b, s, c):
        h.update(np.ascontiguousarray(x).tobytes())
    assert np.array_equal(np.frombuffer(h.digest(), np.uint8), st[p + 'input_sha256']), name
    return b, s, c


def _stable(idx, scores):
    idx = np.asarray(idx, np.int64)
    return idx[np.lexsort((idx, -scores[idx]))] if idx.size else idx


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_oracle_equals_torchvision_per_class_nms():
    """the oracle's keep list is torchvision's _batched_nms_vanilla keep set in the stable (score desc, index asc)
    order, and its score sequence is vanilla's; batched_nms is vanilla above 1000 boxes; the coordinate trick differs
    exactly on the recorded cases"""
    st = _fixture()
    names = [str(n) for n in st['cases']]
    assert len(names) == 10 and list(st['trick_differs']) == ['trick_rounding']
    for name in names:
        b, s, c = _case(st, name)
        got = C.per_class_nms(b, s, c, IOU)
        van = st[name + '/vanilla']
        assert np.array_equal(got, _stable(van, s)), name
        assert np.array_equal(s[got], s[van]), name
        trick = st[name + '/trick']
        assert (set(trick.tolist()) != set(van.tolist())) == (name == 'trick_rounding'), name
        if len(s) > 1000:
            assert np.array_equal(st[name + '/batched'], van), name
    # the properties the crafted cases were made for
    assert np.array_equal(C.per_class_nms(*_case(st, 'identical'), IOU), [0, 1, 2])     # one box per class survives
    assert np.array_equal(C.per_class_nms(*_case(st, 'iou_half'), IOU), [0, 2, 1])      # IoU 0.5 kept, 0.5025 not
    b, s, _ = _case(st, 'one_class')
    assert np.array_equal(C.per_class_nms(b, s, np.zeros(len(s)), IOU),
                          C.O.nms_greedy(torch.from_numpy(b), torch.from_numpy(s), IOU).numpy())
    assert C.per_class_nms(*_case(st, 'empty'), IOU).size == 0


@pytest.mark.parametrize('seed', [0, 1])
def test_per_class_soft_nms_equals_soft_nms_class_by_class(seed):
    b, s, c = C.random_class_candidates(seed, 400, 5, size=200.0, clusters=6, threshold=0.1)
    a = np.random.default_rng(seed).permutation(2000)[:400]
    for method, nt, sigma in (('linear', 0.3, 0.5), ('gaussian', 0.5, 0.5)):
        pa, ps = C.per_class_soft_nms(b, s, c, a, method, nt, sigma, 0.1)
        assert len(pa) > 100
        assert np.array_equal(np.lexsort((pa, -ps)), np.arange(len(pa)))                # (score desc, anchor asc)
        cls_of = dict(zip(a.tolist(), c.tolist()))
        for k in range(5):
            mine = np.array([cls_of[int(v)] == k for v in pa], bool)
            i = np.flatnonzero(c == k)
            wa, ws = S.soft_nms(b[i], s[i], a[i], method, nt, sigma, 0.1)
            assert np.array_equal(pa[mine], wa) and np.array_equal(ps[mine].view(np.uint32), ws.view(np.uint32))


def test_topk_equals_stable_argsort():
    """ties straddling the k-th pair, scores exactly at the threshold (excluded), negative and zero scores"""
    rng = np.random.default_rng(4)
    cls = rng.uniform(-0.2, 1, (300, 7)).astype(np.float32)
    cls[rng.random(cls.shape) < 0.3] = np.float32(0.625)
    cls[rng.random(cls.shape) < 0.05] = np.float32(0.05)
    flat = cls.reshape(-1)
    order = np.argsort(-flat, kind='stable')
    order = order[flat[order] > np.float32(0.05)]
    above, tied = (flat > np.float32(0.625)).sum(), (flat == np.float32(0.625)).sum()
    assert above > 100 and tied > 100
    for k in (1, 17, above + tied // 2, len(order) - 1, len(order), len(order) + 5, 10 ** 6):   # 3rd: k-th is a tie
        assert np.array_equal(C.topk_pairs(cls, 0.05, k), order[:k]), k


def test_python_refuses_bad_class_nms_settings():
    """class_nms and pre_nms_top_k are checked on the host before anything reaches the device (CPU tensors here)"""
    from models import EfficientDet, _ops
    from models._native import EffdetNativeError
    x = torch.zeros(1, 10, 3)
    for kw, what in ((dict(class_nms='class'), 'class_nms'), (dict(class_nms=None), 'class_nms'),
                     (dict(pre_nms_top_k=0), 'pre_nms_top_k'), (dict(pre_nms_top_k=-1), 'pre_nms_top_k'),
                     (dict(pre_nms_top_k=1.5), 'pre_nms_top_k'), (dict(pre_nms_top_k=None), 'pre_nms_top_k'),
                     (dict(class_nms='per_class', pre_nms_top_k=0), 'pre_nms_top_k')):
        with pytest.raises(EffdetNativeError, match=what):
            _ops.detect_batch(x, x, x, 10, 10, 0.05, 0.5, **kw)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    assert (m.class_nms, m.pre_nms_top_k) == ('agnostic', 5000)
    assert m.postprocess() == dict(threshold=0.01, iou_threshold=0.5, nms='hard', sigma=0.5)
    m.class_nms, m.pre_nms_top_k = 'multi_label', 100
    assert m.postprocess() == dict(threshold=0.01, iou_threshold=0.5, nms='hard', sigma=0.5, class_nms='multi_label',
                                   pre_nms_top_k=100)
    for attr, value in (('class_nms', 'perclass'), ('pre_nms_top_k', 0), ('pre_nms_top_k', 1.5),
                        ('pre_nms_top_k', None)):
        setattr(m, attr, value)
        with pytest.raises(EffdetNativeError, match=attr):
            m(torch.zeros(1, 3, 128, 128))
        m.class_nms, m.pre_nms_top_k = 'multi_label', 100
    with pytest.raises(EffdetNativeError, match='class_nms'):
        EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, class_nms='batched')
    assert _ops.candidate_cap(None, x) == 10
    assert _ops.candidate_cap(None, x, 'multi_label', 7) == 7 and _ops.candidate_cap(50, x, 'multi_label') == 30


@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_class_nms_entry_points_refuse_bad_arguments(lib):
    """each refusal returns -1, names the entry point and comes before any device work: the pointers are never
    dereferenced, so these calls run without a GPU"""
    f = 1 << 20

    def refused(rc, name, what=''):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and name in msg and what in msg, (rc, msg)

    ws = lib.effdet_nms_chunked_workspace(2, 1000, 1000)

    def hard(*, p=f, cls=f, B=2, A=2000, npad=2048, cap=1000, chunk=1000, w=f, wb=ws):
        return lib.effdet_nms_batch_chunked_classes(p, p, p, cls, B, A, npad, cap, chunk, 0.5, w, wb, p, p, 0, None)

    for kw, what in ((dict(cls=None), 'null'), (dict(p=None), 'null'), (dict(B=0), 'B='), (dict(npad=1000), 'npad'),
                     (dict(cap=2001, chunk=2001), 'cap'), (dict(chunk=100), 'chunk'), (dict(wb=ws - 1), 'workspace'),
                     (dict(w=f + 8), 'aligned')):
        refused(hard(**kw), 'nms_batch_chunked_classes', what)

    def soft(*, p=f, B=2, cap=1000, method=2, obox=f):
        return lib.effdet_soft_nms_batch_classes(p, p, p, p, p, B, 2000, 2048, cap, method, 0.5, 0.5, 0.05, f, 0,
                                                 p, p, obox, p, 0, None)

    for kw, what in ((dict(p=None), 'null'), (dict(B=65536), 'B='), (dict(cap=0), 'cap'), (dict(method=0), 'method'),
                     (dict(obox=f + 8), 'aligned')):
        refused(soft(**kw), 'soft_nms_batch_classes', what)

    wsb = lib.effdet_detect_topk_workspace(2, 49104, 80, 5000)
    assert wsb == 2 * (2048 * 4 + 32)
    for args, what in (((0, 10, 10, 5), 'B='), ((65536, 10, 10, 5), 'B='), ((1, 10, 10, 0), 'top_k'),
                       ((1, 1 << 26, 64, 5), '2^32'), ((1, 0, 10, 5), 'A=')):
        refused(lib.effdet_detect_topk_workspace(*args), 'detect_topk_workspace', what)

    def topk(*, p=f, B=2, A=49104, K=80, top_k=5000, kpad=8192, w=f, wb=wsb, box=f):
        return lib.effdet_detect_topk_batch(p, p, p, B, A, K, 512.0, 512.0, 0.05, top_k, kpad, w, wb, box, p, p, p, p,
                                            0, None)

    for kw, what in ((dict(p=None), 'null'), (dict(w=None), 'null'), (dict(B=65536), 'B='), (dict(top_k=0), 'top_k'),
                     (dict(A=1 << 26, K=64), '2^32'), (dict(kpad=4096), 'kpad'), (dict(kpad=6000), 'kpad'),
                     (dict(wb=wsb - 1), 'workspace'), (dict(box=f + 4), 'aligned'), (dict(w=f + 8), 'aligned')):
        refused(topk(**kw), 'detect_topk_batch', what)
    # top_k above A*K: k' = A*K sets the smallest kpad
    refused(topk(A=10, K=3, top_k=5000, kpad=16), 'detect_topk_batch', 'kpad')
    assert ctypes.c_int64(lib.effdet_detect_topk_workspace(1, 10, 3, 5000)).value == 2048 * 4 + 32


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device('cuda:0')


def _pack(images, A=None):
    """images: list of (boxes [n,4], scores [n], classes [n], anchors [n]) -> device tensors as
    effdet_detect_candidates_batch leaves them, plus A and npad"""
    A = max([int(a.max()) + 1 for _, _, _, a in images if len(a)] + [1]) if A is None else A
    npad = 1 << (A - 1).bit_length()
    B = len(images)
    rng = np.random.default_rng(5)
    boxes = rng.uniform(0, 50, (B, A, 4)).astype(np.float32)
    scores = np.zeros((B, A), np.float32)
    classes = rng.integers(0, 90, (B, A)).astype(np.int32)
    keys = np.full((B, npad), -1, np.int64)
    count = np.zeros(B, np.int32)
    for b, (bx, sc, cl, an) in enumerate(images):
        boxes[b, an], scores[b, an], classes[b, an] = bx, sc, cl
        order = np.float32(sc).view(np.uint32).astype(np.uint64) ^ np.uint64(0x80000000)   # positive floats only
        k = ((~order & np.uint64(0xffffffff)) << np.uint64(32)) | an.astype(np.uint64)
        keys[b, :len(an)] = np.sort(k).view(np.int64)
        count[b] = len(an)
    t = lambda x: torch.from_numpy(x).to(_dev())                                     # noqa: E731
    return dict(boxes=t(boxes), scores=t(scores), classes=t(classes), keys=t(keys), count=t(count), A=A, npad=npad)


def _run_hard(p, cap, per_class=True):
    from models import _ops
    B, A = p['boxes'].shape[:2]
    o_s = torch.empty((B, cap), device=_dev())
    o_c = torch.empty((B, cap), device=_dev(), dtype=torch.int64)
    o_b = torch.empty((B, cap, 4), device=_dev())
    nk = torch.empty((B,), device=_dev(), dtype=torch.int32)
    _ops._hard_nms(p['boxes'], p['boxes'], p['scores'], p['classes'], p['keys'], p['count'], B, A, p['npad'], cap,
                   IOU, o_s, o_c, o_b, nk, per_class)
    return o_s.cpu().numpy(), o_c.cpu().numpy(), o_b.cpu().numpy(), nk.cpu().numpy()


def _run_soft(p, cap, method, nt, sigma, thr):
    from models import _native as N
    from models import _ops
    B, A = p['boxes'].shape[:2]
    ws_bytes = _ops._soft_nms_workspace(B, cap)
    ws = torch.empty((max(ws_bytes, 16),), device=_dev(), dtype=torch.uint8)
    o_s = torch.empty((B, cap), device=_dev())
    o_c = torch.empty((B, cap), device=_dev(), dtype=torch.int64)
    o_b = torch.empty((B, cap, 4), device=_dev())
    o_n = torch.empty((B,), device=_dev(), dtype=torch.int32)
    N.call('effdet_soft_nms_batch_classes', p['boxes'], N.f32(p['boxes']), N.f32(p['scores']),
           p['classes'].data_ptr(), p['keys'].data_ptr(), p['count'].data_ptr(), B, A, p['npad'], cap,
           _ops.NMS_METHODS[method], nt, sigma, thr, ws.data_ptr(), ws_bytes, N.f32(o_s), o_c.data_ptr(), N.f32(o_b),
           o_n.data_ptr())
    return o_s.cpu().numpy(), o_c.cpu().numpy(), o_b.cpu().numpy(), o_n.cpu().numpy()


def _check(out, images, cap, want_anchors):
    """padded rows of every image equal the oracle's kept anchors (want_anchors(image) -> (anchors, scores))"""
    o_s, o_c, o_b, o_n = out
    for b, (bx, sc, cl, an) in enumerate(images):
        if len(an) > cap:
            assert o_n[b] == -1 and not o_s[b].any() and not o_b[b].any(), b
            continue
        wa, ws = want_anchors(bx, sc, cl, an)
        pos = {int(v): i for i, v in enumerate(an)}
        i = np.asarray([pos[int(v)] for v in wa], np.int64)
        k = len(wa)
        assert o_n[b] == k, (b, o_n[b], k)
        assert np.array_equal(o_s[b, :k].view(np.uint32), np.asarray(ws, np.float32).view(np.uint32)), b
        assert np.array_equal(o_c[b, :k], cl[i]) and np.array_equal(o_b[b, :k].reshape(-1, 4).view(np.uint32),
                                                                   bx[i].reshape(-1, 4).view(np.uint32)), b
        assert not o_s[b, k:].any() and not o_c[b, k:].any() and not o_b[b, k:].any(), b


def _hard_want(bx, sc, cl, an):
    order = np.lexsort((an, -sc))                                    # the candidates in sorted order
    k = order[C.per_class_nms(bx[order], sc[order], cl[order], IOU)]
    return an[k], sc[k]


def _fixture_images():
    st = _fixture()
    rng = np.random.default_rng(9)
    out = []
    for name in (str(n) for n in st['cases']):
        b, s, c = _case(st, name)
        out.append((b, s, c, rng.permutation(8 * max(len(s), 1))[:len(s)].astype(np.int64)))
    return out


@gpu
def test_per_class_hard_nms_equals_oracle_on_fixture_and_chunk_boundaries():
    """every fixture case as one image of a batch; counts 4095, 4096, 4097 and 12 289 around the 4096-candidate NMS
    chunk (the cross step); an image over the cap reports -1; with one class the per-class path equals the agnostic
    one"""
    images = _fixture_images()
    cap = max(len(x[1]) for x in images)
    p = _pack(images)
    _check(_run_hard(p, cap), images, cap, _hard_want)
    for n in (4095, 4096, 4097, 12289):
        A = n + 100
        rng = np.random.default_rng(n)
        imgs = []
        for m, K in ((n, 20), (n + 50, 20), (n, 3)):
            b, s, c = C.random_class_candidates(n + m + K, m, K, size=900.0, clusters=60)
            imgs.append((b, s, c, rng.permutation(A)[:m].astype(np.int64)))
        p = _pack(imgs, A)
        _check(_run_hard(p, n), imgs, n, _hard_want)
        one = [(b, s, np.zeros_like(c), a) for b, s, c, a in imgs]
        p1 = _pack(one, A)
        got, agn = _run_hard(p1, n), _run_hard(p1, n, per_class=False)
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(got, agn)), n


@gpu
@pytest.mark.parametrize('n,cap', [(4096, 4096), (4097, 4097), (8192, 8192), (8193, 8193)])
def test_per_class_soft_nms_equals_oracle(n, cap):
    """per-class Soft-NMS on every fixture case (first parameter set) and on both sides of the shared-memory slice
    capacity boundaries of csrc/soft_nms.cu, both methods"""
    for method, nt, sigma, thr in (('gaussian', 0.5, 0.5, 0.05), ('linear', 0.3, 0.5, 0.05)):
        want = lambda bx, sc, cl, an: C.per_class_soft_nms(bx, sc, cl, an, method, nt, sigma, thr)   # noqa: E731
        if n == 4096:
            images = _fixture_images()
            c0 = max(len(x[1]) for x in images)
            _check(_run_soft(_pack(images), c0, method, nt, sigma, thr), images, c0, want)
        rng = np.random.default_rng(n)
        A = cap + 7
        images = []
        for m, K in ((cap + 5, 20), (0, 20), (n, 20)):
            b, s, c = C.random_class_candidates(n + m, m, K, size=1200.0, clusters=200)
            images.append((b, s, c, rng.permutation(A)[:m].astype(np.int64)))
        _check(_run_soft(_pack(images, A), cap, method, nt, sigma, thr), images, cap, want)


def _topk(cls, threshold, top_k):
    """effdet_detect_topk_batch on cls [B,A,K] (reg zero, anchors fixed) -> NumPy boxes, scores, classes, keys, count"""
    from models import _native as N
    from models import _ops
    B, A, K = cls.shape
    kp = _ops.multi_label_slots(A, K, top_k)
    kpad = 1 << (kp - 1).bit_length()
    reg = torch.zeros((B, A, 4), device=_dev())
    g = torch.arange(A, device=_dev(), dtype=torch.float32)[:, None]
    anchors = torch.cat([g, g, g + 8, g + 16], 1).contiguous()
    boxes = torch.empty((B, kp, 4), device=_dev())
    scores = torch.empty((B, kp), device=_dev())
    classes = torch.empty((B, kp), device=_dev(), dtype=torch.int32)
    keys = torch.empty((B, kpad), device=_dev(), dtype=torch.int64)
    count = torch.empty((B,), device=_dev(), dtype=torch.int32)
    wsb = _ops._topk_workspace(B, A, K, kp)
    ws = torch.empty((wsb // 8,), device=_dev(), dtype=torch.int64)
    N.call('effdet_detect_topk_batch', cls, N.f32(cls), N.f32(reg), N.f32(anchors), B, A, K, 1e6, 1e6,
           float(threshold), kp, kpad, ws.data_ptr(), wsb, N.f32(boxes), N.f32(scores), classes.data_ptr(),
           keys.data_ptr(), count.data_ptr())
    return [t.cpu().numpy() for t in (boxes, scores, classes, keys, count)], anchors.cpu().numpy()


def _check_topk(cls, threshold, top_k):
    (boxes, scores, classes, keys, count), anchors = _topk(cls, threshold, top_k)
    c = cls.cpu().numpy()
    K = c.shape[2]
    for b in range(c.shape[0]):
        p = C.topk_pairs(c[b], threshold, top_k)
        n = len(p)
        assert count[b] == n, (b, count[b], n)
        assert np.array_equal(scores[b, :n].view(np.uint32), c[b].reshape(-1)[p].view(np.uint32)), b
        assert np.array_equal(classes[b, :n], p % K), b
        assert np.array_equal(boxes[b, :n], anchors[p // K]), b                       # zero regression: the anchor
        kb = keys[b].view(np.uint64)
        assert np.array_equal(kb[:n] & np.uint64(0xffffffff), np.arange(n, dtype=np.uint64)), b
        assert np.array_equal(kb[:n] >> np.uint64(32), C.pair_keys(c[b])[p] >> np.uint64(32)), b
        assert np.all(kb[n:] == np.uint64(~np.uint64(0))), b
        assert not scores[b, n:].any() and not classes[b, n:].any() and not boxes[b, n:].any(), b


@gpu
def test_topk_kernel_equals_oracle():
    """counts below, at and above k; k = 1; a run of equal scores straddling the k-th key; scores exactly at the
    threshold (excluded); an image with no pair above the threshold"""
    rng = np.random.default_rng(6)
    A, K = 3000, 9
    c = rng.uniform(0, 1, (5, A, K)).astype(np.float32)
    c[0] = np.where(rng.random((A, K)) < 0.001, c[0], 0.01)                            # ~27 pairs above 0.05
    c[1, :, :] = 0.0
    c[1].reshape(-1)[rng.permutation(A * K)[:100]] = 0.5                              # exactly k = 100 pairs
    c[2][rng.random((A, K)) < 0.3] = np.float32(0.75)                                # ~8100 ties at 0.75
    c[3][rng.random((A, K)) < 0.2] = np.float32(0.05)                                # at the threshold
    c[4] = 0.0
    cls = torch.from_numpy(c).to(_dev())
    for k in (1, 100, 2000, 5000, A * K):
        _check_topk(cls, 0.05, k)


@gpu
def test_topk_kernel_at_d0_512_k80_b32():
    """D0 512x512 (49 104 anchors) with K = 80 at B = 32: 3.9 M pairs per image, seeded scores with ties"""
    g = torch.Generator(device=_dev()).manual_seed(3)
    cls = torch.rand((32, 49104, 80), device=_dev(), generator=g)
    cls[:, ::7, 3] = 0.99
    _check_topk(cls, 0.05, 5000)
    _check_topk(cls[:4], 0.9999, 5000)


def _d0(seed=3, K=20):
    import effdet_oracle as O
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=seed))
    return m.to(_dev()).eval()


def _candidates(cls, reg, anchors, h, w, thr):
    """the device's candidate stage (every anchor decoded) -> NumPy boxes, scores, classes, count, keys"""
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
    cand = _candidates(cls, reg, anchors, h, w, post['threshold'])
    c = cls.cpu().numpy()
    return [C.detect(cand, b, post.get('class_nms', 'agnostic'), post['nms'], post['threshold'],
                     post['iou_threshold'], post['sigma'], post.get('pre_nms_top_k', 5000), c)
            for b in range(cls.shape[0])]


def _same_dets(got, want):
    for b, ((gs, gc, gb), (ws, wc, wb)) in enumerate(zip(got, want)):
        gs, gc, gb = (t.cpu().numpy() for t in (gs, gc, gb))
        assert len(gs) == len(ws), (b, len(gs), len(ws))
        assert np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), b
        assert np.array_equal(gc, wc) and np.array_equal(gb.reshape(-1, 4).view(np.uint32),
                                                         wb.reshape(-1, 4).view(np.uint32)), b


@gpu
@pytest.mark.parametrize('K', [20, 80])
def test_multi_label_and_per_class_on_network_outputs_equal_oracle(K):
    """D0 512x512, seeded weights, B = 4: 'multi_label' at thresholds 0.05 and 0.01 with all three methods, eager and
    at a fixed cap; 'per_class' hard at 0.05; model.detect_batch equals detect_batch"""
    import effdet_oracle as O
    from models import _ops
    m = _d0(K=K)
    x = O.synthetic_batch(4, size=512, seed=8)[0].to(_dev())
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
    runs = [(thr, nms, 'multi_label') for thr in (0.05, 0.01) for nms in ('hard', 'linear', 'gaussian')]
    for thr, nms, mode in runs + [(0.05, 'hard', 'per_class')]:
        m.threshold, m.nms, m.class_nms = thr, nms, mode
        post = m.postprocess()
        want = _oracle_dets(cls, reg, anchors, 512, 512, post)
        _same_dets(_ops.detect_batch(cls, reg, anchors, 512, 512, **post), want)
        fixed = _ops.detect_batch(cls, reg, anchors, 512, 512, cap=cls.shape[1], **post)
        n = fixed.count.tolist()
        if mode == 'multi_label':
            assert fixed.scores.shape[1] == 5000 and max(n) > 0
        _same_dets([(fixed.scores[b, :n[b]], fixed.classes[b, :n[b]], fixed.boxes[b, :n[b]]) for b in range(4)],
                   want)
    m._raw_predictions = lambda images: (cls[:images.shape[0]], reg[:images.shape[0]], anchors)
    with torch.no_grad():
        got = m.detect_batch(x)
    want = _ops.detect_batch(cls, reg, anchors, 512, 512, **m.postprocess())
    assert all(torch.equal(a, b) for g, w in zip(got, want) for a, b in zip(g, w))


@gpu
def test_graphed_detect_in_each_mode_equals_eager():
    """GraphedDetect in each mode replays equal to eager detect_batch; changing class_nms or pre_nms_top_k after
    capture raises; in 'per_class' mode an image over max_candidates reports -1 and is redone eagerly to the same
    rows; the default mode records the same launches as before the class-aware modes existed"""
    import effdet_oracle as O
    from models import _ops
    from models.graph_step import GraphedDetect
    from models._native import EffdetNativeError
    m = _d0()
    m.threshold = 0.05
    x = O.synthetic_batch(4, size=512, seed=8)[0].to(_dev())
    launches = {}
    for mode, nms in (('agnostic', 'hard'), ('per_class', 'hard'), ('per_class', 'gaussian'),
                      ('multi_label', 'hard'), ('multi_label', 'linear')):
        m.class_nms, m.nms = mode, nms
        det = GraphedDetect(m, x, max_candidates=None)
        launches[(mode, nms)] = det.library_launches
        got = det.to_list(det(x))
        want = _ops.detect_batch(det.cls, det.reg, det.anchors, 512, 512, **m.postprocess())
        assert all(torch.equal(a, b) for g, w in zip(got, want) for a, b in zip(g, w)), (mode, nms)
        for attr, value in (('class_nms', 'agnostic' if mode != 'agnostic' else 'per_class'), ('pre_nms_top_k', 77)):
            old = getattr(m, attr)
            setattr(m, attr, value)
            with pytest.raises(EffdetNativeError, match='post-processing settings changed'):
                det(x)
            setattr(m, attr, old)
        del det
    print('library launches per GraphedDetect capture:', launches)
    m.class_nms, m.nms = 'per_class', 'hard'
    probe = GraphedDetect(m, x, max_candidates=None)
    counts = sorted((probe.cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist())
    del probe
    small = GraphedDetect(m, x, max_candidates=max(1, counts[-1] // 2))
    out = small(x)
    assert (out.count == -1).any(), out.count
    want = _ops.detect_batch(small.cls, small.reg, small.anchors, 512, 512, **m.postprocess())
    got = small.to_list(out)
    assert all(torch.equal(a, b) for g, w in zip(got, want) for a, b in zip(g, w))


class _Stub(torch.nn.Module):
    """a detector whose raw outputs are fixed elementwise functions of the pixels, with EfficientDet's post-processing
    settings"""

    def __init__(self, K=4):
        super().__init__()
        from models.module import Anchors
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.K, self.anchors = K, Anchors()
        self.threshold, self.iou_threshold, self.nms, self.soft_nms_sigma = 0.5, 0.5, 'hard', 0.5
        self.class_nms, self.pre_nms_top_k = 'per_class', 5000
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
        self.set_name = 'classnms'

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
@pytest.mark.parametrize('mode', ['per_class', 'multi_label'])
def test_evaluation_in_class_aware_modes_equals_oracles(mode, tmp_path, monkeypatch):
    """evaluate() and evaluate_coco() (batch_size 4: graphed batches and an eager remainder) equal
    tools/voc_eval_oracle.py / tools/coco_eval_oracle.py on the oracle's detections.  Per-class NMS keeps more than
    evaluate_coco's default 1000 records per image here, which the default refuses, naming the capacity that fits."""
    import coco_eval_oracle as CO
    import voc_eval_oracle as V
    from models import evaluation
    K, n = 4, 10
    m = _Stub(K).to(_dev()).eval()
    m.class_nms, m.pre_nms_top_k = mode, 300
    ds = _Data(n, K)
    dets = []
    with torch.no_grad():
        for i in range(n):
            x = ds[i]['img'].permute(2, 0, 1)[None].to(_dev())
            cls, reg, anchors = m._raw_predictions(x)
            dets.append(_oracle_dets(cls, reg, anchors, 256, 256, m.postprocess())[0])
    assert sum(len(d[0]) for d in dets) > 100
    sel = [V.select_detections(s, c, b, ds.scales[i], 0.05, 100, K) for i, (s, c, b) in enumerate(dets)]
    want = V.evaluate(sel, V.get_annotations(ds), K, 0.5)
    got = evaluation.evaluate(ds, m, batch_size=4)
    assert got[0] == want[0], (got[0], want[0])
    assert {c: (float(a), float(k)) for c, (a, k) in got[1].items()} == \
        {c: (float(a), float(k)) for c, (a, k) in want[1].items()}
    anns = []
    for i in range(n):
        for r in ds.annots[i]:
            x1, y1, x2, y2, c = (float(v) for v in r)
            anns.append({'id': len(anns) + 1, 'image_id': ds.image_ids[i], 'category_id': int(c) + 1,
                         'bbox': [x1, y1, x2 - x1, y2 - y1], 'area': (x2 - x1) * (y2 - y1), 'iscrowd': 0})
    inst = {'images': [{'id': i} for i in ds.image_ids], 'categories': [{'id': k + 1} for k in range(K)],
            'annotations': anns}
    ds.coco = CO.COCO(inst)
    results = []
    for i, (s, c, b) in enumerate(dets):
        results += CO.collect(ds.image_ids[i], s, c, b, ds.scales[i], ds.label_to_coco_label)
    want = CO.evaluate(inst, results, ds.image_ids)[0]
    monkeypatch.chdir(tmp_path)
    m.eval()
    if len(results) > 1000 * n:
        with pytest.raises(evaluation.N.EffdetNativeError, match='max_records=%d would' % len(results)):
            evaluation.evaluate_coco(ds, m, batch_size=4)
        m.eval()
    got = evaluation.evaluate_coco(ds, m, batch_size=4, max_records=len(results))
    assert np.array_equal(np.asarray(got), np.asarray(want)), (got, want)
