"""demo.py's per-frame path (Detect.process, demo.py:71-104) on the device: tools/frame_oracle.py against the fixture
pinned to OpenCV and to demo.py's own expressions (tests/golden/make_frame_golden.py), and -- on the GPU --
frame_transform / effdet_frame_transform, frame_boxes / effdet_frame_boxes and GraphedFrameDetect against the oracle,
bit for bit."""
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
import frame_oracle as F  # noqa: E402

G = os.path.join(HERE, 'golden')


def _fixture():
    return np.load(os.path.join(G, 'frame_transform.npz'))


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def _case(st, name):
    p = name + '/'
    sizes = [tuple(int(v) for v in s) for s in st[p + 'sizes']]
    frames = F.synthetic_frames(int(st[p + 'seed'][0]), sizes)
    assert np.array_equal(_sha(np.concatenate([f.reshape(-1) for f in frames])), st[p + 'input_sha256'])
    H, W = (int(v) for v in st[p + 'target'])
    return frames, H, W


def _check(st, name, out):
    p = name + '/'
    assert out.dtype == np.float32 and out.shape[0] == len(st[p + 'sizes'])
    assert np.array_equal(out[:, :, 0, :], st[p + 'first_row']), name
    assert np.array_equal(np.stack([_sha(o) for o in out]), st[p + 'output_sha256']), name


def test_oracle_equals_fixture():
    st = _fixture()
    names = [str(n) for n in st['cases']]
    assert str(st['cv2_version']) == '4.13.0' and len(names) == 12
    geometries = set()
    for name in names:
        frames, H, W = _case(st, name)
        _check(st, name, F.transform(frames, H, W))
        geometries |= {(f.shape[0], f.shape[1], H, W) for f in frames}
    for h, w in [(480, 640), (720, 1280), (1080, 1920), (375, 500), (1024, 1024), (512, 512), (7, 5), (1, 1), (1, 300),
                 (300, 1)]:
        assert (h, w, 512, 512) in geometries, (h, w)
    assert {(480, 640, 384, 640), (720, 1280, 384, 640), (384, 640, 384, 640)} <= geometries


def test_oracle_equals_demo_arithmetic():
    """boxes and scores as demo.py's own expressions compute them under the installed NumPy (>= 2: float32), with rows
    where the NumPy 1.x float64 reading truncates differently and scores where round(100 * s) differs"""
    st = _fixture()
    b_in, hw, size = st['boxes/in'], st['boxes/frame_hw'], st['boxes/size_hw']
    for reading, key in ((False, 'boxes/out'), (True, 'boxes/out_numpy1')):
        got = np.concatenate([F.frame_boxes(b[None], [0], [0], h, s, float64=reading)[0] for b, h, s in zip(b_in, hw, size)])
        assert np.array_equal(got, st[key]), key
    assert (st['boxes/out'] != st['boxes/out_numpy1']).any(axis=1).sum() >= 8
    s_in = st['scores/in']
    assert np.array_equal(F.frame_boxes(np.zeros((len(s_in), 4)), np.zeros(len(s_in)), s_in, (1, 1))[2], st['scores/out'])
    assert (np.round(s_in.astype(np.float64) * 100).astype(np.int32) != st['scores/out']).any()


def test_oracle_equals_cv2_sweep():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.RandomState(5)
    for _ in range(24):
        h, w = int(rng.randint(1, 900)), int(rng.randint(1, 900))
        H, W = int(rng.randint(1, 800)), int(rng.randint(1, 800))
        img = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
        for opt in (True, False):
            cv2.setUseOptimized(opt)
            assert np.array_equal(cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR), F.resize_u8(img, H, W)), \
                (h, w, H, W, opt)
    cv2.setUseOptimized(True)


def test_oracle_resize_rules():
    """the branches of resize_u8 on hand-checkable inputs"""
    img = np.arange(4 * 6 * 3, dtype=np.uint8).reshape(4, 6, 3)
    assert np.array_equal(F.resize_u8(img, 4, 6), img)                              # same size: a copy
    s = img.astype(int)
    want = (s[2, 4] + s[2, 5] + s[3, 4] + s[3, 5] + 2) >> 2                          # exact 2x: rounded 2x2 mean
    assert np.array_equal(F.resize_u8(img, 2, 3)[1, 2], want)
    flat = np.full((3, 5, 3), 77, np.uint8)                                          # a constant stays constant
    assert (F.resize_u8(flat, 11, 2) == 77).all()


def test_ctypes_mirrors_match_header():
    import re
    from models import _native
    hdr = open(os.path.join(REPO, 'include', 'effdet_b200.h')).read()
    for name in ('effdet_frame_transform', 'effdet_frame_boxes'):
        decl = re.search(r'int %s\(([^)]*)\);' % name, hdr).group(1)
        params = [p.strip() for p in decl.split(',')]
        argtypes = _native.SIGNATURES[name]
        assert len(params) == len(argtypes), name
        for p, t in zip(params, argtypes):
            if p in ('const float* mean3', 'const float* std3'):
                assert t is ctypes.POINTER(ctypes.c_float), (name, p)
            elif '*' in p or p.startswith('effdet_stream_t'):
                assert t is ctypes.c_void_p
            else:
                assert p.startswith('int ') and t is ctypes.c_int, (name, p)


def test_argument_refusals_before_launch():
    """the entry points, frame_transform and GraphedFrameDetect refuse bad arguments before anything touches the
    device, so these calls run without a GPU"""
    from models import _native
    from models._native import EffdetNativeError
    from models.graph_step import GraphedFrameDetect
    from models.pipeline import frame_transform
    _native.build()
    lib = _native.load()

    def err():
        return lib.effdet_last_error().decode()

    fake = 1 << 20
    f3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    assert lib.effdet_frame_transform(fake, fake, None, fake, 1, 512, 512, f3, f3, 0, None) == -1 and 'null' in err()
    assert lib.effdet_frame_transform(fake, fake, fake, fake, 0, 512, 512, f3, f3, 0, None) == -1 and 'B=0' in err()
    assert lib.effdet_frame_transform(fake, fake, fake, fake, 1, 0, 512, f3, f3, 0, None) == -1 and 'H=0' in err()
    assert lib.effdet_frame_transform(fake, fake, fake, fake, 1, 512, 70000, f3, f3, 0, None) == -1 and 'W=70000' in err()
    assert lib.effdet_frame_transform(fake, fake, fake, fake, 1, 512, 512, None, f3, 0, None) == -1 and 'null' in err()
    assert lib.effdet_frame_boxes(fake, fake, fake, fake, None, 1, 8, 512, 512, fake, fake, 0, None) == -1
    assert 'null' in err()
    assert lib.effdet_frame_boxes(fake, fake, fake, fake, fake, 0, 8, 512, 512, fake, fake, 0, None) == -1
    assert 'B=0' in err()
    assert lib.effdet_frame_boxes(fake, fake, fake, fake, fake, 1, 0, 512, 512, fake, fake, 0, None) == -1
    assert 'C=0' in err()
    assert lib.effdet_frame_boxes(fake, fake, fake + 4, fake, fake, 1, 8, 512, 512, fake, fake, 0, None) == -1
    assert 'aligned' in err()
    assert lib.effdet_frame_boxes(fake, fake, fake, fake, fake, 1, 8, 0, 512, fake, fake, 0, None) == -1
    assert 'H=0' in err()

    ok = np.zeros((4, 5, 3), np.uint8)
    bad = [np.zeros((4, 5, 3), np.float32), np.zeros((4, 5, 2), np.uint8), np.zeros((4, 5), np.uint8),
           np.zeros((0, 5, 3), np.uint8), np.zeros((4, 0, 3), np.uint8)]
    for im in bad:
        with pytest.raises(EffdetNativeError, match='uint8'):
            frame_transform([ok, im])
        with pytest.raises(EffdetNativeError, match='uint8'):
            GraphedFrameDetect(None, [ok, im])
    for empty in ([], np.zeros((1, 4, 5, 3), np.uint8)):
        with pytest.raises(EffdetNativeError, match='non-empty list'):
            frame_transform(empty)
    with pytest.raises(EffdetNativeError, match='height'):
        frame_transform([ok], height=0)


# ------------------------------------------------------------------------------------------------------------- GPU

def _model(num_classes=20):
    import effdet_oracle as O
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', num_classes=num_classes, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=num_classes, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=5))
    return m.cuda().eval()


def _rows_of(out, b, hw, H, W):
    """the oracle's contract 3 on frame b of padded Detections `out` (the device's own network outputs)"""
    n = int(out.count[b])
    return F.frame_boxes(out.boxes[b, :n].cpu().numpy(), out.classes[b, :n].cpu().numpy(),
                         out.scores[b, :n].cpu().numpy(), hw, (H, W))


@pytest.mark.gpu
def test_frame_transform_bit_exact():
    from models.pipeline import frame_transform
    st = _fixture()
    for name in [str(n) for n in st['cases']]:
        frames, H, W = _case(st, name)
        out = frame_transform(frames, H, W)
        assert out.is_cuda and tuple(out.shape) == (len(frames), 3, H, W)
        got = out.cpu().numpy()
        _check(st, name, got)
        assert np.array_equal(got, F.transform(frames, H, W)), name


@pytest.mark.gpu
def test_frame_boxes_bit_exact():
    """effdet_frame_boxes on crafted padded detections: a frame with no rows, a frame whose every row of C is kept, the
    fixture's truncation and rounding splits, a padding frame (h = 0) and an overflowed frame (count -1)"""
    from models import _ops
    from models.pipeline import frame_boxes
    st = _fixture()
    s_in = st['scores/in']
    for H, W in {tuple(int(v) for v in s) for s in st['boxes/size_hw']}:
        sel = (st['boxes/size_hw'] == [H, W]).all(axis=1)
        b_in, hws = st['boxes/in'][sel], st['boxes/frame_hw'][sel]
        frames = [tuple(int(v) for v in hw) for hw in np.unique(hws, axis=0)]
        B, C = len(frames) + 4, 64
        scores = np.zeros((B, C), np.float32)
        classes = np.zeros((B, C), np.int64)
        boxes = np.zeros((B, C, 4), np.float32)
        count = np.zeros((B,), np.int32)
        hw = np.zeros((B, 2), np.int32)
        rng = np.random.RandomState(H + W)
        for b, fhw in enumerate(frames):
            rows = b_in[(hws == fhw).all(axis=1)][:C]
            n = len(rows)
            boxes[b, :n], count[b], hw[b] = rows, n, fhw
            scores[b, :n] = rng.choice(s_in, n)
            classes[b, :n] = rng.randint(0, 20, n)
        full, empty, pad, over = len(frames), len(frames) + 1, len(frames) + 2, len(frames) + 3
        boxes[full] = rng.rand(C, 4) * [W, H, W, H]
        scores[full] = s_in[:C]
        classes[full] = np.arange(C) % 90
        count[full], hw[full] = C, (720, 1280)
        count[empty], hw[empty] = 0, (480, 640)
        count[pad], hw[pad], boxes[pad] = C, (0, 0), 7.0               # padding frame: rows present, count 0
        count[over], hw[over] = -1, (480, 640)
        t = lambda a: torch.from_numpy(a).cuda()                       # noqa: E731
        det = _ops.Detections(t(scores), t(classes), t(boxes), t(count))
        rows, counts = frame_boxes(det, t(hw), H, W)
        counts = counts.cpu().numpy()
        want = count.copy()
        want[pad] = 0
        assert np.array_equal(counts, want)
        rows = rows.cpu().numpy()
        for b in range(B):
            n = max(int(counts[b]), 0)
            xy, lab, sc = F.frame_boxes(boxes[b, :n], classes[b, :n], scores[b, :n], tuple(hw[b]), (H, W))
            assert np.array_equal(rows[b, :n, :4], xy) and np.array_equal(rows[b, :n, 4], lab) and \
                np.array_equal(rows[b, :n, 5], sc), (H, W, b)
        # the rows the fixture pinned to demo.py itself
        for b, fhw in enumerate(frames):
            m = (hws == fhw).all(axis=1)
            n = min(int(m.sum()), C)
            assert np.array_equal(rows[b, :n, :4], st['boxes/out'][sel][m][:n]), (H, W, fhw)


def _frames(seed, sizes):
    return F.synthetic_frames(seed, sizes)


@pytest.mark.gpu
@pytest.mark.parametrize('bcap', [1, 8])
def test_graphed_frame_detect(bcap):
    """the replay's input is the oracle's transform of the frames (padding frames zero), and its rows are the oracle's
    contract 3 applied to that replay's own detections; short calls and new frame sizes replay without recapture"""
    from models.graph_step import GraphedFrameDetect
    from models._native import EffdetNativeError
    m = _model()
    sizes = [(480, 640), (720, 1280), (375, 500), (1080, 1920), (1, 300), (512, 512), (7, 5), (1024, 1024)][:bcap]
    det = GraphedFrameDetect(m, _frames(50, sizes))
    calls = [_frames(51, sizes), _frames(52, sizes[::-1])]
    if bcap > 1:
        calls += [_frames(53, [(600, 800), (300, 1)]), _frames(54, [(333, 500)] * (bcap - 1))]
    else:
        calls += [_frames(53, [(400, 600)])]
    for frames in calls:
        res = det(frames)
        B = len(frames)
        assert len(res) == B
        x = det.static_images.cpu().numpy()
        assert np.array_equal(x[:B], F.transform(frames, 512, 512))
        assert not x[B:].any()
        counts = det.out.count.cpu().numpy()
        for b, (boxes, labels, scores) in enumerate(res):
            assert counts[b] >= 0 and len(boxes) == counts[b] > 0
            assert boxes.dtype == np.int32 and labels.dtype == np.int64 and scores.dtype == np.int32
            xy, lab, sc = _rows_of(det.out, b, frames[b].shape[:2], 512, 512)
            assert np.array_equal(boxes, xy) and np.array_equal(labels, lab) and np.array_equal(scores, sc), b
            assert (boxes[:, 2] <= frames[b].shape[1]).all() and (boxes[:, 3] <= frames[b].shape[0]).all()
    with pytest.raises(EffdetNativeError, match='capacity'):
        det(_frames(55, sizes + [(4, 4)]))
    with pytest.raises(EffdetNativeError, match='capacity'):
        det(_frames(56, [(det.byte_capacity // 3000 + 1, 1000)]))           # one frame, more bytes than fit


@pytest.mark.gpu
def test_graphed_frame_detect_matches_demo_call():
    """against demo.py's own call: eager model(x) at B = 1 on the oracle-transformed frame, then the oracle's rescale.
    Two passes of the network differ in the last bits (fp32 atomics), so rows are matched per label with integer boxes
    and scores within 1; the share of matched rows is printed (DESIGN.md section 8 item 5 records it)."""
    from models.graph_step import GraphedFrameDetect
    m = _model()
    frame = _frames(60, [(720, 1280)])
    det = GraphedFrameDetect(m, frame)
    boxes, labels, scores = det(frame)[0]
    with torch.no_grad():
        s, c, b = m(torch.from_numpy(F.transform(frame)).cuda())
    e_xy, e_lab, e_sc = F.frame_boxes(b.cpu().numpy(), c.cpu().numpy(), s.cpu().numpy(), (720, 1280))
    matched = 0
    for lab in np.union1d(labels, e_lab):
        g = np.concatenate([boxes[labels == lab], scores[labels == lab, None]], axis=1).astype(np.int64)
        e = np.concatenate([e_xy[e_lab == lab], e_sc[e_lab == lab, None]], axis=1).astype(np.int64)
        used = np.zeros(len(e), bool)
        for row in g:
            ok = np.flatnonzero(~used & (np.abs(e - row) <= 1).all(axis=1))
            if len(ok):
                used[ok[0]] = True
                matched += 1
    n, ne = len(boxes), len(e_xy)
    print('demo call: %d graph rows, %d eager rows, %d matched within 1 (%.4f)' % (n, ne, matched, matched / max(n, ne)))
    assert n > 0 and abs(n - ne) <= max(1, n // 100) and matched >= 0.99 * max(n, ne)


@pytest.mark.gpu
def test_graphed_frame_detect_overflow_redone_eagerly():
    """with max_candidates below the candidate count every frame overflows the captured NMS; its rows are then the
    eager NMS of the replay's own network outputs, rescaled as demo.py does"""
    from models import _ops
    from models.graph_step import GraphedFrameDetect
    m = _model()
    frames = _frames(57, [(480, 640), (375, 500)])
    det = GraphedFrameDetect(m, frames, max_candidates=256)
    res = det(frames)
    assert (det.out.count.cpu().numpy() == -1).all()
    for b, (boxes, labels, scores) in enumerate(res):
        s, c, bx = _ops.detect_batch(det.cls[b:b + 1], det.reg[b:b + 1], det.anchors, 512, 512, m.threshold,
                                     m.iou_threshold)[0]
        xy, lab, sc = F.frame_boxes(bx.cpu().numpy(), c.cpu().numpy(), s.cpu().numpy(), frames[b].shape[:2])
        assert len(boxes) > 256 and np.array_equal(boxes, xy) and np.array_equal(labels, lab) and \
            np.array_equal(scores, sc), b
