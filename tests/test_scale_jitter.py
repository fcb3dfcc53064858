"""Scale-jitter training augmentation: RawCollater(scale_jitter=(lo, hi)) draws a common size L and a window (y0, x0) per
image on the host, and the raw graphed training step resizes at L and crops to S x S on the device
(effdet_resize_crop_normalize_pad), with the boxes shifted, clamped and filtered (effdet_collate_pack_annots_crop).

CPU: tools/jitter_oracle.py against the reference-pinned fixture tests/golden/pipeline_jitter.npz, the draws, the
jittered blob's layout, and the refusals (ranges, evaluation, the new entry points' arguments).
GPU: both crop kernels against the oracle bit for bit (fixture cases, seeded batches, box edge cases), scale_jitter=(1, 1)
against the unjittered raw path, and GraphedTrainStep on jittered batches against the oracle and against the tensor
capacity-mode step over a 2-worker epoch."""
import hashlib
import math
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from test_graphed_train_loop import D0_MEDIAN, D0_WORST, _d0, _rel
from test_raw_batches import FAKE, _Dataset, _model, _samples, _Samples

import effdet_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
import jitter_oracle as J  # noqa: E402
import resize_oracle as R  # noqa: E402


def _dev():
    return torch.device('cuda:0')


def _fixture():
    return np.load(os.path.join(HERE, 'golden', 'pipeline_jitter.npz'))


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def _case(st, name):
    """a fixture case's inputs (regenerated from its seed, every third row labelled -1) and recorded geometry"""
    p = name + '/'
    sizes = [tuple(int(v) for v in s) for s in st[p + 'sizes']]
    images, annots = R.synthetic_batch(int(st[p + 'seed'][0]), sizes, [int(n) for n in st[p + 'n_boxes']])
    for a in annots:
        a[2::3, 4] = -1
    assert np.array_equal(_sha(np.concatenate([im.reshape(-1) for im in images])), st[p + 'input_sha256'])
    return dict(images=images, annots=annots, flips=[bool(f) for f in st[p + 'flips']], S=int(st[p + 'common'][0]),
                enc=255 if bool(st[p + 'voc'][0]) else None, resized=st[p + 'resized'], crops=st[p + 'crops'],
                scales=st[p + 'scales'], L=st[p + 'L'], drawn=st[p + 'drawn_L'])


def _case_raw(c, capacity=None):
    """a jittered RawBatch carrying a fixture case's recorded geometry (no draws)"""
    from models.pipeline import _assemble
    B = len(c['images'])
    counts = np.array([a.shape[0] for a in c['annots']], dtype=np.int32)
    raw = _assemble(B, c['S'], c['enc'], np.array([im.shape[:2] for im in c['images']], dtype=np.int32),
                    c['resized'], np.array(c['flips'], dtype=np.uint8), c['scales'], counts,
                    np.concatenate(c['annots']), c['images'], crops=c['crops'])
    return raw if capacity is None else raw.at_capacity(capacity)


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_oracle_equals_golden_fixture():
    """every fixture case: the raise of L and the Resizer geometry are pipeline's, and the oracle's windows (digest,
    first two rows, last row inside the resized image) and packed boxes are the reference chain's"""
    from models.pipeline import min_common_size, resizer_geometry
    st = _fixture()
    for name in [str(n) for n in st['cases']]:
        c = _case(st, name)
        S, B = c['S'], len(c['images'])
        wins, kept = [], []
        for b, im in enumerate(c['images']):
            h, w = im.shape[:2]
            L = max(int(c['drawn'][b]), min_common_size(h, w))
            assert L == c['L'][b], name
            scale, rh, rw = resizer_geometry(h, w, L)
            assert scale == c['scales'][b] and [rh, rw] == c['resized'][b].tolist(), name
            y0, x0 = (int(v) for v in c['crops'][b])
            wins.append(J.crop_image(im, c['flips'][b], rh, rw, y0, x0, S, c['enc']))
            kept.append(J.crop_boxes(c['annots'][b], c['flips'][b], w, scale, y0, x0, S))
        wins = np.stack(wins)
        p = name + '/'
        assert np.array_equal(_sha(wins), st[p + 'images_sha256']), name
        assert np.array_equal(wins[:, :, :2, :], st[p + 'top_rows']), name
        last = [wins[b, :, max(min(int(c['resized'][b][0]) - int(c['crops'][b][0]), S), 1) - 1] for b in range(B)]
        assert np.array_equal(np.stack(last), st[p + 'last_rows']), name
        table, counts = J.pack(kept, B, st[p + 'annots'].shape[1])
        assert np.array_equal(table, st[p + 'annots']) and np.array_equal(counts, st[p + 'counts']), name


def _count_randint(monkeypatch):
    calls = []
    real = np.random.randint

    def randint(*a, **k):
        calls.append(a)
        return real(*a, **k)

    monkeypatch.setattr(np.random, 'randint', randint)
    return calls


def test_draws_are_in_range_three_per_image_and_reproducible(monkeypatch):
    """seeded np.random: L in [L_lo, L_hi] (or raised), 0 <= y0 <= max(rh - S, 0) and likewise x0; exactly three
    randint calls per image in sample order, the same draws as replaying them by hand; the same seed gives the same
    blob"""
    from models.pipeline import RawCollater, jitter_range, min_common_size, resizer_geometry
    S = 512
    sizes = [(375, 500), (480, 640), (500, 375), (7, 5), (1, 300), (2000, 30), (333, 500)]
    samples = _samples(31, sizes, [2] * len(sizes))
    col = RawCollater(S, pixel_scale=255, scale_jitter=(0.1, 2.0))
    L_lo, L_hi = jitter_range(S, 0.1, 2.0)
    assert (L_lo, L_hi) == (52, 1024)
    calls = _count_randint(monkeypatch)
    np.random.seed(5)
    raw = col(samples)
    assert len(calls) == 3 * len(sizes)
    assert raw.jitter and raw.section('header')[6] == 1
    resized, crops = raw.section('resized_hw').numpy(), raw.section('crops').numpy()
    np.random.seed(5)
    for b, (h, w) in enumerate(sizes):                              # the contract's draws, replayed
        L = max(int(np.random.randint(L_lo, L_hi + 1)), min_common_size(h, w))
        scale, rh, rw = resizer_geometry(h, w, L)
        y0 = np.random.randint(0, max(rh - S, 0) + 1)
        x0 = np.random.randint(0, max(rw - S, 0) + 1)
        assert [rh, rw] == resized[b].tolist() and [y0, x0] == crops[b].tolist() and raw.scales[b] == scale, b
        assert L_lo <= L <= L_hi or L == min_common_size(h, w)
        assert 0 <= y0 <= max(rh - S, 0) and 0 <= x0 <= max(rw - S, 0)
    np.random.seed(5)
    assert torch.equal(col(samples).blob, raw.blob)
    many = RawCollater(S, scale_jitter=(0.1, 2.0))
    Ls = []
    for seed in range(40):
        np.random.seed(seed)
        r = many(samples[:2])
        Ls += r.section('resized_hw').numpy().max(axis=1).tolist()
        c, rhw = r.section('crops').numpy(), r.section('resized_hw').numpy()
        assert (c >= 0).all() and (c <= np.maximum(rhw - S, 0)).all()
    assert min(Ls) >= L_lo and max(Ls) <= L_hi and max(Ls) > S > min(Ls)


def test_raise_of_L():
    """min_common_size is the smallest L at which the Resizer keeps both sides >= 1 (brute force); an image whose
    aspect ratio exceeds every drawable L is resized at that L and never refused"""
    from models.pipeline import RawCollater, min_common_size, resizer_geometry
    for h, w in [(1, 1), (1, 2), (2, 1), (1, 700), (700, 1), (3, 2000), (900, 2), (10, 10), (375, 500), (7, 5000)]:
        L = min_common_size(h, w)
        assert min(resizer_geometry(h, w, L)[1:]) >= 1 and (L == 1 or min(resizer_geometry(h, w, L - 1)[1:]) < 1)
    col = RawCollater(512, scale_jitter=(0.1, 0.5))
    np.random.seed(3)
    raw = col(_samples(32, [(1, 700), (900, 2), (100, 100)], [1, 1, 1]))
    assert raw.section('resized_hw').tolist()[:2] == [[1, 700], [450, 1]]
    assert 52 <= raw.section('resized_hw')[2, 0] <= 256
    assert raw.section('crops').tolist()[1] == [0, 0] and 0 <= raw.section('crops')[0, 1] <= 700 - 512


def test_unit_jitter_is_the_common_size_and_no_offset():
    """scale_jitter=(1, 1): every image at L = S, windows at (0, 0); the blob is the unjittered one plus the crops
    section and header[6] = 1"""
    from models.pipeline import RawCollater, raw_layout
    samples = _samples(33, [(375, 500), (500, 375), (1, 300), (640, 480)], [3, 0, 1, 2], flips=[1, 0, 1, 0])
    plain = RawCollater(512, 255)(samples)
    unit = RawCollater(512, 255, scale_jitter=(1, 1))(samples)
    assert not unit.section('crops').any()
    for name in ('offsets', 'hw', 'resized_hw', 'flips', 'scales', 'row_offsets'):
        if name != 'offsets':
            assert torch.equal(unit.section(name), plain.section(name)), name
    assert np.array_equal(unit.scales, plain.scales)
    h_u, h_p = unit.section('header').tolist(), plain.section('header').tolist()
    assert h_u[6] == 1 and h_p[6] == 0 and h_u[:6] == h_p[:6]
    po, _ = raw_layout(4, plain.rows, plain.nbytes)
    uo, _ = raw_layout(4, unit.rows, unit.nbytes, jitter=True)
    assert torch.equal(unit.blob[uo['rows']:], plain.blob[po['rows']:])


def test_dataloader_workers_draw_differently():
    from models.pipeline import RawCollater
    samples = _samples(34, [(375, 500)] * 2, [1, 1]) * 4
    loader = torch.utils.data.DataLoader(_Dataset(samples), batch_size=2, shuffle=False, num_workers=2,
                                         collate_fn=RawCollater(256, scale_jitter=(0.1, 2.0)))
    got = [(r.section('resized_hw').tolist(), r.section('crops').tolist()) for r in loader]
    assert len(got) == 4 and got[0] != got[1], got                  # batches 0 and 1 come from different workers


def test_jittered_blob_layout_and_round_trips(monkeypatch):
    """16-byte aligned sections with crops right before rows; at_capacity, pin_memory and pickling keep the flag and
    the crops; the sections before crops sit where an unjittered blob has them"""
    from models.pipeline import RawBatch, RawCollater, raw_layout
    for cap, rows, nbytes in [(1, 0, 3), (3, 7, 1001), (32, 411, 375 * 500 * 3 * 32)]:
        off, total = raw_layout(cap, rows, nbytes, jitter=True)
        plain, _ = raw_layout(cap, rows, nbytes)
        assert all(v % 16 == 0 for v in off.values()) and total % 16 == 0
        assert off['row_offsets'] < off['crops'] < off['rows'] <= off['pixels']
        assert off['rows'] >= off['crops'] + 8 * cap and off['rows'] == raw_layout(cap, 0, 0, jitter=True)[0]['rows']
        assert all(off[k] == plain[k] for k in plain if k not in ('rows', 'pixels'))
    np.random.seed(8)
    samples = _samples(35, [(37, 51), (8, 300), (120, 90)], [2, 0, 5], flips=[1, 0, 1])
    raw = RawCollater(64, pixel_scale=255, scale_jitter=(0.5, 2.0))(samples)
    assert raw.section('crops').any()
    big = raw.at_capacity(6)
    assert big.jitter and big.section('header')[6] == 1 and big.capacity == 6
    assert torch.equal(big.section('crops')[:3], raw.section('crops')) and not big.section('crops')[3:].any()
    for name in ('hw', 'resized_hw', 'flips', 'scales'):
        assert torch.equal(big.section(name)[:3], raw.section(name)), name
    bo, _ = raw_layout(6, raw.rows, raw.nbytes, jitter=True)
    ro, _ = raw_layout(3, raw.rows, raw.nbytes, jitter=True)
    assert torch.equal(big.blob[bo['rows']:bo['rows'] + 40 * raw.rows], raw.blob[ro['rows']:ro['rows'] + 40 * raw.rows])
    monkeypatch.setattr(torch.Tensor, 'pin_memory', lambda self: self.clone())   # no CUDA here: the copy, not the pin
    pinned = raw.pin_memory()
    assert pinned.jitter and torch.equal(pinned.blob, raw.blob)
    back = pickle.loads(pickle.dumps(raw))
    assert isinstance(back, RawBatch) and back.jitter and torch.equal(back.blob, raw.blob)
    col = pickle.loads(pickle.dumps(RawCollater(384, scale_jitter=(0.1, 2.0))))
    assert col.scale_jitter == (0.1, 2.0) and col.S == 384


@pytest.mark.parametrize('bad', [(0, 1), (-0.5, 1), (1.5, 1.0), (float('nan'), 1), (0.1, float('inf')),
                                 (float('-inf'), 1), (1,), (0.1, 0.5, 2.0), 'ab', 1.0, (0.5, 200.0)])
def test_bad_ranges_are_refused(bad):
    from models._native import EffdetNativeError
    from models.pipeline import RawCollater
    with pytest.raises(EffdetNativeError, match='scale_jitter'):
        RawCollater(512, scale_jitter=bad)


def test_evaluation_refuses_a_jittering_collater(monkeypatch):
    """evaluate() and evaluate_coco() refuse a collater with scale_jitter before they start a loader or touch the
    model"""
    from models import _native as N
    from models import evaluation
    from models.pipeline import RawCollater

    def no_loader(*a, **k):
        raise AssertionError('a loader was started')

    monkeypatch.setattr(torch.utils.data, 'DataLoader', no_loader)
    col = RawCollater(512, pixel_scale=255, scale_jitter=(0.1, 2.0))
    with pytest.raises(N.EffdetNativeError, match='evaluate: .*scale_jitter'):
        evaluation.evaluate(object(), object(), collater=col, num_workers=2)
    with pytest.raises(N.EffdetNativeError, match='evaluate_coco: .*scale_jitter'):
        evaluation.evaluate_coco(object(), object(), collater=col, num_workers=2)


@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_crop_entries_refuse_bad_arguments_before_any_launch(lib):
    import ctypes
    err = lambda: lib.effdet_last_error().decode()                       # noqa: E731
    m3 = (ctypes.c_double * 3)(0, 0, 0)

    def resize(ptrs=None, B=2, S=64, ps=1, mean=m3, std=m3):
        return lib.effdet_resize_crop_normalize_pad(*(ptrs or [FAKE] * 7), B, S, ps, mean, std, 0, None)

    for i in range(6):                                                   # flip (index 5) may be null
        ptrs = [FAKE] * 7
        ptrs[i if i < 5 else 6] = None
        assert resize(ptrs) == -1 and 'resize_crop_normalize_pad: bad arguments' in err(), i
    for bad in (dict(B=0), dict(B=65536), dict(S=0), dict(S=65536), dict(mean=None), dict(std=None)):
        assert resize(**bad) == -1 and 'resize_crop_normalize_pad: bad arguments' in err(), bad
    assert resize(ps=2) == -1 and 'pixel_scale 2' in err()

    def pack(ptrs=None, Bcap=4, Gcap=8):
        return lib.effdet_collate_pack_annots_crop(*(ptrs or [FAKE] * 9), Bcap, Gcap, 0, None)

    for i in range(9):
        ptrs = [FAKE] * 9
        ptrs[i] = None
        assert pack(ptrs) == -1 and 'collate_pack_annots_crop: null argument' in err(), i
    for bad in (dict(Bcap=0), dict(Bcap=65536), dict(Gcap=0), dict(Gcap=-1), dict(Gcap=(1 << 31) // 5 + 1)):
        assert pack(**bad) == -1 and 'collate_pack_annots_crop: capacity' in err(), bad
    if not torch.cuda.is_available():                                    # valid arguments: only the device fails
        assert resize() < 0 and 'resize_crop' not in err() and 'cuda' in err().lower()
        assert pack() < 0 and 'collate_pack_annots_crop' not in err() and 'cuda' in err().lower()


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level
# ------------------------------------------------------------------------------------------------------------------

def _device_unpack(raw, Gcap):
    """both crop launches on the device copy of raw -> (images, table, counts) as NumPy, outputs pre-filled with NaN /
    -7 so every element must be written"""
    from models.pipeline import launch_raw_pack, launch_raw_resize
    blob = raw.blob.to(_dev())
    cap = raw.capacity
    imgs = torch.full((cap, 3, raw.S, raw.S), float('nan'), device=_dev())
    table = torch.full((cap, Gcap, 5), float('nan'), device=_dev())
    counts = torch.full((1 + cap,), -7, dtype=torch.int32, device=_dev())
    launch_raw_resize(imgs, blob, cap, raw.pixel_scale, raw.jitter)
    launch_raw_pack(blob, cap, table, counts, raw.jitter)
    torch.cuda.synchronize()
    return imgs.cpu().numpy(), table.cpu().numpy(), counts.cpu().numpy()


def _bits_equal(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.gpu
def test_crop_kernels_equal_oracle_on_fixture_cases():
    st = _fixture()
    for name in [str(n) for n in st['cases']]:
        c = _case(st, name)
        raw = _case_raw(c)
        Gcap = st[name + '/annots'].shape[1]
        imgs, table, counts = _device_unpack(raw, Gcap)
        assert np.array_equal(_sha(imgs), st[name + '/images_sha256']), name
        assert _bits_equal(table, st[name + '/annots']) and np.array_equal(counts, st[name + '/counts']), name
        o_imgs, o_table, o_counts = J.from_raw(raw, Gcap)
        assert _bits_equal(imgs, o_imgs) and _bits_equal(table, o_table) and np.array_equal(counts, o_counts), name


@pytest.mark.gpu
@pytest.mark.parametrize('S,enc', [(512, 255), (1536, None)])
def test_crop_kernels_equal_oracle_on_seeded_batches(S, enc):
    """seeded RawCollater(scale_jitter=(0.1, 2.0)) batches of B = 8 VOC / COCO-sized images with flips in Bcap = 10:
    images, table and counts bit for bit; the two padding slots are exact +0"""
    from models.pipeline import RawCollater
    rng = np.random.RandomState(S)
    sizes = [[(375, 500), (500, 375), (480, 640), (640, 480)][i % 4] for i in range(8)]
    samples = _samples(S + 1, sizes, [int(n) for n in rng.randint(0, 9, size=8)], flips=rng.randint(0, 2, size=8),
                       neg_every=4)
    np.random.seed(S + 2)
    raw = RawCollater(S, pixel_scale=enc, scale_jitter=(0.1, 2.0))(samples).at_capacity(10)
    L = raw.section('resized_hw').numpy()[:8].max(axis=1)
    print('S=%d drawn L: %s, windows %s' % (S, L.tolist(), raw.section('crops')[:8].tolist()))
    assert (L > S).any() and (L < S).any()
    imgs, table, counts = _device_unpack(raw, 16)
    o_imgs, o_table, o_counts = J.from_raw(raw, 16)
    assert _bits_equal(imgs, o_imgs)
    assert _bits_equal(table, o_table) and np.array_equal(counts, o_counts)
    assert (imgs[8:] == 0).all() and not np.signbit(imgs[8:]).any()


@pytest.mark.gpu
def test_unit_jitter_equals_the_unjittered_raw_path():
    """scale_jitter=(1, 1) with boxes inside their images: images, table and counts equal RawCollater without jitter,
    bit for bit, through the crop launches against the unjittered ones"""
    from models.pipeline import RawCollater
    samples = _samples(36, [(375, 500), (500, 375), (480, 640), (1, 300), (512, 512), (1024, 768)], [3, 4, 0, 1, 5, 2],
                       flips=[1, 0, 1, 1, 0, 1], neg_every=3)
    for enc in (255, None):
        plain = RawCollater(512, enc)(samples).at_capacity(8)
        unit = RawCollater(512, enc, scale_jitter=(1, 1))(samples).at_capacity(8)
        a, b = _device_unpack(plain, 8), _device_unpack(unit, 8)
        for x, y in zip(a, b):
            assert x.shape == y.shape and np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                                         y.view(np.uint32) if y.dtype == np.float32 else y)


@pytest.mark.gpu
def test_crop_pack_kernel_box_edge_cases():
    """rows straddling each window edge, wholly outside it, reaching zero area after the clamp, labelled -1; an image
    that loses every row; an image that fills Gcap exactly; the crop pack kernel == the oracle, bit for bit"""
    from models.pipeline import _assemble
    S, Gcap = 100, 9
    # image 0: 400 x 400 at L = 200 (scale 0.5), window (50, 60): x in [60, 160), y in [50, 150) in resized pixels
    edge = [[100, 200, 180, 260, 1],        # straddles the left edge
            [300, 200, 360, 260, 2],        # straddles the right edge
            [200, 80, 260, 120, 3],         # straddles the top edge
            [200, 280, 260, 340, 4],        # straddles the bottom edge
            [0, 0, 110, 90, 5],             # wholly outside, above left
            [330, 310, 400, 400, 6],        # wholly outside, below right
            [100, 200, 120, 260, 7],        # x range left of the window: zero width after the clamp
            [200, 320, 260, 340, 8],        # below the window: zero height after the clamp
            [200, 200, 260, 260, -1],       # inside, label -1
            [200, 200, 260, 260, 9],        # inside
            [120, 100, 320, 300, 10]]       # covers the window: clamped to [0, S] on every side
    outside = [[0, 0, 10, 10, 1], [390, 0, 400, 10, 2], [150, 150, 180, 180, -1]]     # image 1 loses every row
    full = [[10 * i, 10 * i, 10 * i + 50, 10 * i + 50, i] for i in range(Gcap)]       # image 2 keeps Gcap rows
    rows = [np.array(r, dtype=np.float64) for r in (edge, outside, full)]
    rows[0][:4, :4] += 0.3                                                              # non-integral coordinates
    sizes = np.array([[400, 400], [400, 400], [200, 200]], dtype=np.int32)
    imgs = [np.zeros((h, w, 3), np.uint8) for h, w in sizes]
    for flips in ([0, 0, 0], [1, 1, 1]):
        raw = _assemble(4, S, None, sizes, np.array([[200, 200], [200, 200], [200, 200]], np.int32),
                        np.array(flips, np.uint8), np.array([0.5, 0.5, 1.0]), np.array([len(r) for r in rows], np.int32),
                        np.concatenate(rows), imgs, crops=np.array([[50, 60], [50, 60], [0, 0]], np.int32))
        got = _device_unpack(raw, Gcap)[1:]
        want = J.from_raw(raw, Gcap)[1:]
        assert _bits_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), flips
        if not flips[0]:
            assert got[1].tolist() == [3, 6, 0, Gcap, 0], got[1]
            assert got[0][0, :6, 4].tolist() == [1, 2, 3, 4, 9, 10] and got[0][0, 5, :4].tolist() == [0, 0, S, S]


# ------------------------------------------------------------------------------------------------------------------
# GPU, graphed steps
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_graphed_step_on_jittered_batches_equals_oracle():
    """a step built on a jittered batch: after each replay (new draws, a pinned batch, a short batch) its static
    images, annotations and counts equal the oracle on that batch's recorded geometry; built once, never recaptured"""
    from models.graph_step import GraphedTrainStep
    from models.pipeline import RawCollater
    m = _model(seed=81)
    col = RawCollater(256, pixel_scale=255, scale_jitter=(0.1, 2.0))
    pool = _samples(82, [(375, 500), (500, 375), (480, 640), (300, 200), (90, 400)], [3, 0, 12, 5, 1],
                    flips=[1, 0, 1, 0, 1], neg_every=4)
    np.random.seed(83)
    step = GraphedTrainStep(m, col(pool[:4]), max_annotations=16, warmup=1)
    graph = step.graph
    for i, batch in enumerate([pool[:4], pool[1:5], pool[2:4], pool[:4]]):
        raw = col(batch)
        if i == 1:
            raw = raw.pin_memory()
        step(raw)
        torch.cuda.synchronize()
        o_imgs, o_table, o_counts = J.from_raw(raw, 16, Bcap=4)
        assert _bits_equal(step.static_images.cpu().numpy(), o_imgs), i
        assert _bits_equal(step.static_annots.cpu().numpy(), o_table), i
        assert np.array_equal(step.static_counts.cpu().numpy(), o_counts), i
    assert step.graph is graph


@pytest.mark.gpu
def test_jitter_mismatch_and_detection_are_refused_without_launches():
    from models import _native as N
    from models.graph_step import GraphedRawDetect, GraphedTrainStep
    from models.pipeline import RawCollater
    from test_raw_batches import _eval_model
    samples = _samples(84, [(100, 120), (120, 100)], [2, 1])
    plain, jit = RawCollater(128), RawCollater(128, scale_jitter=(0.5, 1.5))
    md, _ = _eval_model(0.3)
    launches = N.launch_count()
    with pytest.raises(N.EffdetNativeError, match='GraphedRawDetect takes unjittered raw batches'):
        GraphedRawDetect(md, jit(samples))
    assert N.launch_count() == launches
    # the detector first: building it invalidates the weight caches that a step built without an optimizer replays
    det = GraphedRawDetect(md, plain(samples))
    m = _model(seed=85)
    steps = {False: GraphedTrainStep(m, plain(samples), max_annotations=4, warmup=1),
             True: GraphedTrainStep(m, jit(samples), max_annotations=4, warmup=1)}
    torch.cuda.synchronize()
    launches = N.launch_count()
    with pytest.raises(N.EffdetNativeError, match='unjittered raw batches, got a batch that is scale-jittered; rebuild'):
        steps[False](jit(samples))
    with pytest.raises(N.EffdetNativeError, match='scale-jittered raw batches, got a batch that is unjittered; rebuild'):
        steps[True](plain(samples))
    with pytest.raises(N.EffdetNativeError, match='GraphedRawDetect takes unjittered raw batches'):
        det(jit(samples))
    assert N.launch_count() == launches
    assert float(steps[True](jit(samples))) >= 0


# The epoch below replays training on test_raw_batches' epoch data with the paper's jitter range (0.1, 2.0).  Two runs
# of the SAME step on the SAME inputs differ by the fp32 atomic order of the backward, and what that becomes after a few updates
# depends on the learning rate: on an H100, tensor step against tensor step, lr 1e-3 reached a loss error of 1.2e-3
# (losses of the late batches grow to 10^2 and amplify it) and lr 1e-4 an update median of 7e-3, each past its bound;
# at lr 5e-4 six runs stayed below 9.0e-5 (loss), 9.2e-4 (update median) and 4.5e-2 (worst update).
LR, JITTER, LOADER_SEED = 5e-4, (0.1, 2.0), 0


def _jittered_epoch(lr, jitter, loader_seed, k=2, floor=False, ds=None):
    """D0 256^2, Bcap 4, Gcap 64, FusedClipAdamW(lr) with k: a DataLoader(num_workers=2, collate_fn=RawCollater(256,
    255, scale_jitter=jitter), pin_memory=True, generator seeded with loader_seed, so every worker's np.random and hence
    every draw is the same on every run) feeding one raw step, then the tensor capacity-mode step fed the oracle's
    images and tables of the same batches -> the comparison's figures"""
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    from models.pipeline import RawCollater
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=86)
    ds = _Samples(23, seed=52) if ds is None else ds
    torch.cuda.init()                                                   # the loader's workers fork after CUDA init

    def run(batches):
        m = _d0(sd)
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        opt = FusedClipAdamW(m.parameters(), lr=lr, max_norm=0.1)
        losses, raws, graphs = [], [], []
        opt.zero_grad()
        if batches is None:
            loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, num_workers=2, pin_memory=True,
                                                 collate_fn=RawCollater(256, pixel_scale=255, scale_jitter=jitter),
                                                 generator=torch.Generator().manual_seed(loader_seed))
            step = None
            for idx, raw in enumerate(loader):
                assert raw.blob.is_pinned() and raw.jitter
                if step is None:
                    step = GraphedTrainStep(m, raw, optimizer=opt, max_annotations=64)
                graphs.append(step.graph)
                losses.append(float(step(raw, update=(idx + 1) % k == 0)))
                raws.append(raw)
        else:
            step = GraphedTrainStep(m, *batches[0], optimizer=opt, max_annotations=64)
            for idx, (images, ann) in enumerate(batches):
                losses.append(float(step(images, ann, update=(idx + 1) % k == 0)))
        torch.cuda.synchronize()
        counts = {int(s['step']) for s in opt.state_dict()['state'].values()}
        return {n: p.detach() - p0[n] for n, p in m.named_parameters()}, losses, counts, raws, graphs

    upd_r, loss_r, steps_r, raws, graphs = run(None)
    batches = []
    for raw in raws:
        imgs, table, _ = J.from_raw(raw, 64)
        batches.append((torch.from_numpy(imgs[:raw.B]).to(_dev()), torch.from_numpy(table[:raw.B]).to(_dev())))
    upd_t, loss_t, steps_t, _, _ = run(batches)

    def errs(upd, loss):
        e = sorted(_rel(upd[n], upd_t[n]) for n in upd_t if float(upd_t[n].abs().max()) > 0)
        return e, max(abs(a - b) / abs(b) for a, b in zip(loss, loss_t) if b != 0)

    e, loss_err = errs(upd_r, loss_r)
    if floor:                                                           # the tensor step against itself
        upd_2, loss_2, _, _, _ = run(batches)
        e2, l2 = errs(upd_2, loss_2)
        print('tensor vs tensor: update rel err median %.2e worst %.2e; loss rel err %.2e' % (e2[len(e2) // 2], e2[-1], l2))
    print('jittered epoch lr %g jitter %s: windows %s; losses %s vs tensor %s; %d updated tensors, update rel err '
          'median %.2e worst %.2e; loss rel err %.2e'
          % (lr, jitter, [r.section('crops').tolist() for r in raws], ['%.5f' % v for v in loss_r],
             ['%.5f' % v for v in loss_t], len(e), e[len(e) // 2], e[-1], loss_err))
    return dict(raws=raws, graphs=graphs, loss_err=loss_err, n=len(e), med=e[len(e) // 2], worst=e[-1],
                steps=(steps_r, steps_t))


@pytest.mark.gpu
def test_jittered_epoch_with_workers_matches_the_tensor_capacity_step():
    """a 2-worker jittered epoch (_jittered_epoch) through one raw step, never recaptured, against the tensor
    capacity-mode step on the oracle's tensors of the same batches (sizes 4 x 5, 3): per-step losses within 1e-3,
    updates within the D0 bounds of test_dataloader_epoch_with_workers_matches_the_tensor_capacity_step, equal step
    counts.  The loader is seeded, so the draws are fixed; what differs between runs is only the fp32 atomic order, whose
    effect the tensor step against itself shows (printed as the noise floor)."""
    r = _jittered_epoch(LR, JITTER, LOADER_SEED, floor=True)
    assert [b.B for b in r['raws']] == [4, 4, 4, 4, 4, 3] and r['raws'][1].rows == 0
    assert all(g is r['graphs'][0] for g in r['graphs'])
    assert len({tuple(map(tuple, b.section('crops').tolist())) for b in r['raws']}) > 1
    assert r['loss_err'] < 1e-3 and not math.isnan(r['loss_err'])
    assert r['n'] > 250 and r['med'] < D0_MEDIAN and r['worst'] < D0_WORST
    assert r['steps'][0] == r['steps'][1]
