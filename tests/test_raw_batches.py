"""Raw batches: DataLoader workers collate decoded uint8 samples into one CUDA-free host blob (pipeline.RawCollater ->
RawBatch), and the graphed steps run the Normalizer -> Augmenter flip -> Resizer -> collater chain and the annotation
packing at the head of their graphs.

CPU: the blob's geometry, scales and sections against resizer_geometry and the fixture of test_pipeline_resize.py, the
refusals against DeviceCollater's, pickling and DataLoader workers, and the new entry point's argument checks.
GPU: effdet_collate_pack_annots against effdet_collate_annots + effdet_pack_annots bit for bit; GraphedTrainStep on raw
batches against DeviceCollater + the tensor capacity-mode step; GraphedRawDetect inside evaluate() / evaluate_coco()
against the unchanged functions on datasets that run the host chain."""
import ctypes
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O
from test_graphed_train_loop import D0_MEDIAN, D0_WORST, _d0, _rel
from test_pipeline_resize import _case, _fixture
from test_ragged_train_batches import _eager

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
import resize_oracle as R  # noqa: E402

FAKE = 1 << 20                                               # aligned non-null "pointer"; never dereferenced


def _dev():
    return torch.device('cuda:0')


def _samples(seed, sizes, counts, flips=None, K=20, neg_every=0):
    """decoded samples as a dataset yields them: uint8 [h,w,3] images, float64 [n,5] boxes inside each image (label -1
    on every neg_every-th row, when set), optional flips"""
    images, annots = R.synthetic_batch(seed, sizes, counts)
    out = []
    for b, (im, a) in enumerate(zip(images, annots)):
        a = a.copy()
        a[:, 4] %= K
        if neg_every:
            a[1::neg_every, 4] = -1
        s = dict(img=im, annot=a)
        if flips is not None:
            s['flip'] = bool(flips[b])
        out.append(s)
    return out


class _Dataset(torch.utils.data.Dataset):
    def __init__(self, samples):
        self.samples = samples

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_raw_collater_geometry_and_scales_match_resizer():
    """every fixture case: hw, resized_hw and the scales are resizer_geometry's (and the fixture's scales), the flips,
    rows and pixels are the samples', and the byte offsets point at each image"""
    from models.pipeline import RawCollater, raw_layout, resizer_geometry
    st = _fixture()
    for name in [str(n) for n in st['cases']]:
        images, annots, flips, S, enc = _case(st, name)
        raw = RawCollater(S, pixel_scale=enc)([dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)])
        B = len(images)
        assert raw.B == raw.capacity == B and raw.S == S and raw.pixel_scale == enc
        geo = [resizer_geometry(im.shape[0], im.shape[1], S) for im in images]
        assert np.array_equal(raw.section('hw').numpy(), [im.shape[:2] for im in images])
        assert np.array_equal(raw.section('resized_hw').numpy(), [g[1:] for g in geo])
        assert np.array_equal(raw.section('scales').numpy(), [g[0] for g in geo])
        assert np.array_equal(raw.scales, st[name + '/scales']) and raw.scales.dtype == np.float64
        assert raw.section('flips').tolist() == [int(f) for f in flips]
        assert raw.section('header').tolist()[:6] == [B, raw.nbytes, raw.rows, B, S, enc or 1]
        assert raw.counts.tolist() == [a.shape[0] for a in annots]
        off, total = raw_layout(B, raw.rows, raw.nbytes)
        assert raw.blob.numel() == total and raw.blob.dtype == torch.uint8
        a = raw.blob.numpy()
        rows = a[off['rows']:off['rows'] + 40 * raw.rows].view(np.float64).reshape(-1, 5)
        assert np.array_equal(rows, np.concatenate(annots))
        assert raw.section('row_offsets').tolist() == np.concatenate([[0], np.cumsum(raw.counts)]).tolist()
        for b, im in enumerate(images):
            o = int(raw.section('offsets')[b])
            assert np.array_equal(a[o:o + im.size], im.reshape(-1))


def test_raw_collater_refuses_what_device_collater_refuses():
    from models._native import EffdetNativeError
    from models.pipeline import DeviceCollater, RawCollater
    ok = np.zeros((4, 5, 3), np.uint8)
    box = np.zeros((0, 5))
    bad = [np.zeros((4, 5, 3), np.float32), np.zeros((4, 5, 2), np.uint8), np.zeros((4, 5), np.uint8),
           np.zeros((0, 5, 3), np.uint8), np.zeros((4, 0, 3), np.uint8), np.zeros((1, 700, 3), np.uint8)]
    cases = [[dict(img=ok, annot=box), dict(img=im, annot=box)] for im in bad] + [[dict(img=ok, annot=box, scale=1.0)]]
    for samples in cases:
        msgs = []
        for col in (DeviceCollater(512, resize=True, pixel_scale=255), RawCollater(512, pixel_scale=255)):
            with pytest.raises(EffdetNativeError) as e:
                col(samples)
            msgs.append(str(e.value).split(': ', 1)[1])
        assert msgs[0] == msgs[1], msgs
    with pytest.raises(EffdetNativeError, match='pixel_scale'):
        RawCollater(512, pixel_scale=256)


def test_blob_sections_are_aligned_and_round_trip():
    """16-byte aligned sections; at_capacity(B + 3) keeps every section and zeroes the unused entries; pickling keeps
    the blob and the host facts"""
    from models.pipeline import RawBatch, RawCollater, raw_layout
    for cap, rows, nbytes in [(1, 0, 3), (3, 7, 1001), (32, 411, 375 * 500 * 3 * 32), (65535, 1, 1)]:
        off, total = raw_layout(cap, rows, nbytes)
        assert all(v % 16 == 0 for v in off.values()) and total % 16 == 0
        assert total >= off['pixels'] + nbytes and off['pixels'] >= off['rows'] + 40 * rows
    samples = _samples(3, [(37, 51), (8, 300), (120, 90)], [2, 0, 5], flips=[1, 0, 1])
    raw = RawCollater(256, pixel_scale=255)(samples)
    big = raw.at_capacity(6)
    assert big.capacity == 6 and big.B == 3 and np.array_equal(big.scales, raw.scales)
    for name in ('hw', 'resized_hw', 'flips', 'scales'):
        assert torch.equal(big.section(name)[:3], raw.section(name)) and not big.section(name)[3:].any(), name
    assert torch.equal(big.section('row_offsets')[:4], raw.section('row_offsets'))
    assert not big.section('offsets')[3:].any() and big.section('header').tolist()[:4] == [3, raw.nbytes, 7, 6]
    for b, s in enumerate(samples):
        o = int(big.section('offsets')[b])
        assert np.array_equal(big.blob.numpy()[o:o + s['img'].size], s['img'].reshape(-1))
    back = pickle.loads(pickle.dumps(raw))
    assert isinstance(back, RawBatch) and torch.equal(back.blob, raw.blob)
    assert back.counts.tolist() == [2, 0, 5] and back.nbytes == raw.nbytes and back.S == 256 and back.pixel_scale == 255
    assert pickle.loads(pickle.dumps(RawCollater(384))).S == 384


def _epoch_samples(n=14, seed=11):
    rng = np.random.RandomState(seed)
    sizes = [(int(rng.randint(60, 400)), int(rng.randint(60, 400))) for _ in range(n)]
    counts = [int(c) for c in rng.randint(0, 9, size=n)]
    counts[5] = 37
    return _samples(seed, sizes, counts, flips=rng.randint(0, 2, size=n))


def test_dataloader_workers_yield_the_same_batches():
    from models.pipeline import RawCollater
    ds = _Dataset(_epoch_samples())
    got = {}
    for workers in (0, 2):
        loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, num_workers=workers,
                                             collate_fn=RawCollater(256))
        got[workers] = list(loader)
    assert [r.B for r in got[0]] == [4, 4, 4, 2]
    for a, b in zip(got[0], got[2]):
        assert torch.equal(a.blob, b.blob) and np.array_equal(a.counts, b.counts) and np.array_equal(a.scales, b.scales)


@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_collate_pack_refuses_bad_arguments_before_any_launch(lib):
    def call(ptrs=None, Bcap=4, Gcap=8):
        return lib.effdet_collate_pack_annots(*(ptrs or [FAKE] * 8), Bcap, Gcap, 0, None)

    err = lambda: lib.effdet_last_error().decode()                       # noqa: E731
    for i in range(8):
        ptrs = [FAKE] * 8
        ptrs[i] = None
        assert call(ptrs) == -1 and 'collate_pack_annots' in err() and 'null' in err(), i
    for bad in (dict(Bcap=0), dict(Bcap=65536), dict(Gcap=0), dict(Gcap=-1), dict(Gcap=(1 << 31) // 5 + 1)):
        assert call(**bad) == -1 and 'collate_pack_annots' in err(), bad
    if not torch.cuda.is_available():                                    # valid arguments: only the device fails
        assert call() < 0 and 'collate_pack_annots' not in err() and 'cuda' in err().lower()


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('counts,flips,Bcap,Gcap', [
    ([3, 0, 7, 1], [1, 0, 0, 1], 4, 7),                       # flips, an empty image, G = Gcap
    ([5, 2], [0, 1], 6, 9),                                   # B < Bcap
    ([0, 0, 0], [1, 0, 1], 3, 1),                             # no rows at all
    ([300, 40, 2], [1, 1, 0], 5, 300),                        # more rows than a CTA, G = Gcap
    ([12] * 8, [0, 1] * 4, 8, 256)])
def test_pack_kernel_equals_collate_then_pack(counts, flips, Bcap, Gcap):
    """effdet_collate_pack_annots on the device copy of a raw batch == DeviceCollater(resize=True)'s table (collate_annots
    with the Resizer scales) packed by effdet_pack_annots, bit for bit; -1 labels on every 3rd row exercise the drop"""
    from models import _ops
    from models.pipeline import DeviceCollater, RawCollater, launch_raw_pack
    rng = np.random.RandomState(sum(counts) + Bcap)
    sizes = [(int(rng.randint(20, 700)), int(rng.randint(20, 700))) for _ in counts]
    samples = _samples(len(counts) * 7 + Gcap, sizes, counts, flips=flips, neg_every=3)
    _, ann = DeviceCollater(512, 'cuda:0', resize=True)(samples)
    want = torch.full((Bcap, Gcap, 5), float('nan'), device=_dev())
    want_c = torch.full((1 + Bcap,), -7, dtype=torch.int32, device=_dev())
    _ops.pack_annotations(ann, want, want_c)
    raw = RawCollater(512)(samples).at_capacity(Bcap)
    blob = raw.blob.to(_dev())
    got = torch.full((Bcap, Gcap, 5), float('nan'), device=_dev())
    got_c = torch.full((1 + Bcap,), -7, dtype=torch.int32, device=_dev())
    launch_raw_pack(blob, Bcap, got, got_c)
    assert torch.equal(got_c, want_c), (got_c, want_c)
    assert torch.equal(got, want)
    assert int(got_c[0]) == len(counts) and not got_c[1 + len(counts):].any()
    if max(counts) > 1:                                                   # control: unflipped boxes differ
        plain = RawCollater(512)([dict(s, flip=False) for s in samples]).at_capacity(Bcap)
        launch_raw_pack(plain.blob.to(_dev()), Bcap, got, got_c)
        assert not torch.equal(got, want) or not any(flips)


# ------------------------------------------------------------------------------------------------------------------
# GPU, graphed steps
# ------------------------------------------------------------------------------------------------------------------

def _model(seed=43, train=True):
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    return _d0(O.init_state_dict(cfg, seed=seed))


@pytest.mark.gpu
def test_raw_step_static_images_equal_device_collater():
    """every fixture case, both encodings: a raw step built for B + 1 images and called on the case's B images holds
    DeviceCollater(resize=True)'s images and packed annotations bit for bit, and exact zeros for the padding image"""
    from models import _ops
    from models.graph_step import GraphedTrainStep
    from models.pipeline import DeviceCollater, RawCollater
    st = _fixture()
    m = _model(seed=7)
    for name in [str(n) for n in st['cases']]:
        images, annots, flips, S, enc = _case(st, name)
        samples = [dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)]
        B = len(samples)
        col = RawCollater(S, pixel_scale=enc)
        step = GraphedTrainStep(m, col(samples + samples[:1]), max_annotations=64, warmup=1)
        step(col(samples))
        torch.cuda.synchronize()
        imgs, ann = DeviceCollater(S, 'cuda:0', resize=True, pixel_scale=enc)(samples)
        assert torch.equal(step.static_images[:B], imgs), name
        assert bool((step.static_images[B:] == 0).all()) and not torch.signbit(step.static_images[B:]).any(), name
        want = torch.empty_like(step.static_annots)
        want_c = torch.empty_like(step.static_counts)
        _ops.pack_annotations(ann, want, want_c)
        assert torch.equal(step.static_annots, want) and torch.equal(step.static_counts, want_c), name
        del step
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_raw_graph_launches_and_sync_free_step():
    """the raw graph records the tensor capacity-mode graph's launches + 2 (resize and pack); a step(raw_batch) after
    construction runs under set_sync_debug_mode('error'), pinned or not, full or short"""
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    from models.pipeline import DeviceCollater, RawCollater
    m = _model(seed=8)
    samples = _samples(9, [(300, 200), (256, 256), (90, 400), (250, 260)], [3, 0, 12, 1], flips=[1, 0, 0, 1])
    imgs, ann = DeviceCollater(256, 'cuda:0', resize=True)(samples)
    opt = FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1)
    tensor = GraphedTrainStep(m, imgs, ann, optimizer=opt, max_annotations=16)
    n_tensor = tensor.library_launches
    del tensor
    torch.cuda.empty_cache()
    col = RawCollater(256)
    opt = FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1)           # an optimizer binds to one graph
    step = GraphedTrainStep(m, col(samples), optimizer=opt, max_annotations=16)
    print('library launches: tensor capacity mode %d, raw %d' % (n_tensor, step.library_launches))
    assert step.library_launches == n_tensor + 2
    batches = [col(samples).pin_memory(), col(samples[1:3]).pin_memory(), col(samples), col(samples[:1])]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for i, raw in enumerate(batches):
            step(raw, update=i % 2 == 1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert int(step.static_counts[0]) == 1 and bool((step.static_images[1:] == 0).all())


@pytest.mark.gpu
def test_raw_batches_that_do_not_fit_are_refused_without_side_effects():
    from models import _native as N
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    from models.pipeline import RawCollater
    m = _model(seed=10)
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    col = RawCollater(128)
    example = col(_samples(12, [(100, 120), (120, 100)], [3, 5]))
    with pytest.raises(N.EffdetNativeError, match='max_annotations=5 or more'):
        GraphedTrainStep(m, example, optimizer=opt, max_annotations=4)
    with pytest.raises(N.EffdetNativeError, match='needs max_annotations'):
        GraphedTrainStep(m, example, optimizer=opt)
    step = GraphedTrainStep(m, example, optimizer=opt, max_annotations=8)
    assert step.raw['max_bytes'] == 2 * 120 * 100 * 3
    step(example, update=True)
    torch.cuda.synchronize()
    G = opt._graph

    def state():
        return [t.clone() for t in [step.static_images, step.static_annots, step.static_counts, step.raw['blob'],
                                    G['step'], G['lr'], G['update']] + [p.detach() for p in m.parameters()]
                + [v for st in opt.state.values() for v in st.values() if torch.is_tensor(v)]]

    before = state()
    launches = N.launch_count()
    refusals = [(col(_samples(13, [(50, 60)] * 3, [1, 1, 1])), 'capacity of 2 images'),
                (col(_samples(14, [(200, 121)], [1])), 'max_bytes=72600 or more'),
                (col(_samples(15, [(40, 40), (30, 30)], [9, 0])), 'max_annotations=9 or more'),
                (RawCollater(160)(_samples(16, [(40, 40)], [1])), 'common size 128'),
                (RawCollater(128, 255)(_samples(16, [(40, 40)], [1])), 'pixel_scale')]
    for raw, msg in refusals:
        with pytest.raises(N.EffdetNativeError, match=msg):
            step(raw, update=False)
    with pytest.raises(N.EffdetNativeError, match='step\\(raw_batch'):
        step(example, torch.zeros(1))
    torch.cuda.synchronize()
    assert N.launch_count() == launches and G['update_host'] == 1
    for a, b in zip(before, state()):
        assert torch.equal(a, b)
    loss = step(col(_samples(17, [(60, 70)], [2])), update=True)         # a batch of one still runs after them
    assert float(loss) > 0 and int(step.static_counts[0]) == 1


class _Samples(torch.utils.data.Dataset):
    """a seeded in-memory dataset of decoded samples (what workers would decode from JPEGs)"""

    def __init__(self, n, seed):
        rng = np.random.RandomState(seed)
        sizes = [(int(rng.randint(120, 400)), int(rng.randint(120, 400))) for _ in range(n)]
        counts = [int(c) for c in rng.randint(0, 12, size=n)]
        counts[4:8] = [0, 0, 0, 0]                                       # batch 1: no annotations at all
        counts[2] = 60
        self.samples = _samples(seed, sizes, counts, flips=rng.randint(0, 2, size=n))

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]


@pytest.mark.gpu
def test_dataloader_epoch_with_workers_matches_the_tensor_capacity_step():
    """D0 256^2, Bcap 4, Gcap 64, FusedClipAdamW with k = 2: a DataLoader(num_workers=2, collate_fn=RawCollater(256, 255),
    pin_memory=True) started after CUDA is initialised, feeding the raw step, against the tensor capacity-mode step fed
    DeviceCollater output of the same samples; batch sizes 4, 4, 4, 4, 4, 3, the second without annotations.  The bounds
    of test_dataloader_shaped_epoch_matches_eager_drop_in; control: the eager loop with the tail averaged over Bcap, whose
    losses exceed the loss bound and whose updates sit at least 5x further from the reference than the raw loop's."""
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    from models.pipeline import DeviceCollater, RawCollater
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=51)
    ds = _Samples(23, seed=52)
    k = 2
    dcol = DeviceCollater(256, 'cuda:0', resize=True, pixel_scale=255)
    tensor_batches = [dcol([ds[i] for i in range(i0, min(len(ds), i0 + 4))]) for i0 in range(0, len(ds), 4)]
    assert torch.cuda.is_initialized()

    def run(mode):
        m = _d0(sd)
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        losses = []
        if mode == 'raw':
            loader = torch.utils.data.DataLoader(ds, batch_size=4, shuffle=False, num_workers=2,
                                                 collate_fn=RawCollater(256, pixel_scale=255), pin_memory=True)
            step = None
            opt.zero_grad()
            for idx, raw in enumerate(loader):
                assert raw.blob.is_pinned()
                if step is None:
                    step = GraphedTrainStep(m, raw, optimizer=opt, max_annotations=64)
                losses.append(float(step(raw, update=(idx + 1) % k == 0)))
        elif mode == 'tensor':
            step = GraphedTrainStep(m, *tensor_batches[0], optimizer=opt, max_annotations=64)
            opt.zero_grad()
            for idx, (images, ann) in enumerate(tensor_batches):
                losses.append(float(step(images, ann, update=(idx + 1) % k == 0)))
        else:
            losses = _eager(m, opt, tensor_batches, k, tail_scale=3 / 4)
        torch.cuda.synchronize()
        steps = {int(s['step']) for s in opt.state_dict()['state'].values()}
        return {n: p.detach() - p0[n] for n, p in m.named_parameters()}, losses, steps

    upd_t, loss_t, steps_t = run('tensor')
    upd_r, loss_r, steps_r = run('raw')
    upd_c, loss_c, _ = run('control')

    def errs(upd):
        e = sorted(_rel(upd[n], upd_t[n]) for n in upd_t if float(upd_t[n].abs().max()) > 0)
        return e[len(e) // 2], e[-1], len(e)

    def loss_err(ls):
        return max(abs(a - b) / abs(b) for a, b in zip(ls, loss_t) if b != 0)

    med, worst, n = errs(upd_r)
    print('raw epoch: losses %s vs tensor %s; %d updated tensors, update rel err median %.2e worst %.2e; loss rel err '
          '%.2e; control loss err %.2e, update median %.2e' % (['%.5f' % v for v in loss_r], ['%.5f' % v for v in loss_t],
                                                              n, med, worst, loss_err(loss_r), loss_err(loss_c),
                                                              errs(upd_c)[0]))
    assert len(loss_r) == len(loss_t) == 6 and loss_r[1] == loss_t[1] == 0.0
    assert loss_err(loss_r) < 1e-3
    assert n > 250 and med < D0_MEDIAN and worst < D0_WORST
    assert steps_r == steps_t
    assert loss_err(loss_c) > 1e-3 and errs(upd_c)[0] > 5 * med


# ------------------------------------------------------------------------------------------------------------------
# GPU, evaluation
# ------------------------------------------------------------------------------------------------------------------

def _eval_images(n, seed, high=256):
    """uint8 images in [0, high) whose sizes force the byte-capacity rebuild: the first batch of 4 is small, the second
    large"""
    rng = np.random.RandomState(seed)
    sizes = [(int(rng.randint(80, 140)), int(rng.randint(80, 140))) for _ in range(4)]
    sizes += [(int(rng.randint(200, 420)), int(rng.randint(200, 420))) for _ in range(n - 4)]
    return [rng.randint(0, high, size=s + (3,)).astype(np.uint8) for s in sizes]


class _VOCSet:
    """the VOC generator interface; raw=True yields decoded samples, raw=False what Normalizer + Resizer yield"""

    def __init__(self, images, annotations, K, S, pixel_scale, raw):
        self.images, self.annotations, self.K, self.S, self.pixel_scale, self.raw = images, annotations, K, S, \
            pixel_scale, raw

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        im = self.images[i]
        if self.raw:
            return {'img': im, 'annot': self.annotations[i] if self.annotations else np.zeros((0, 5))}
        scale, rh, rw = R.resizer_geometry(im.shape[0], im.shape[1], self.S)
        new = np.zeros((self.S, self.S, 3))
        new[:rh, :rw] = R.resize_linear(R.normalize(im, self.pixel_scale), rh, rw)
        return {'img': torch.from_numpy(new.astype(np.float32)), 'scale': scale}

    def load_annotations(self, i):
        return self.annotations[i]

    def num_classes(self):
        return self.K

    def label_to_name(self, label):
        return 'class%d' % label


def _eval_model(threshold):
    from models import EfficientDet
    K = 80
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=1, mode='wellcond'))
    m = m.to(_dev()).eval()
    m.threshold = threshold
    return m, K


def _gap(scores):
    """a score in the middle of a wide gap between neighbouring scores (every detection, when there are few)"""
    sc = np.unique(scores)
    assert sc.size > 0
    if sc.size < 10:
        return float(sc[0]) - 1.0
    lo, hi = int(0.3 * sc.size), int(0.7 * sc.size)
    j = lo + int(np.argmax(np.diff(sc[lo:hi])))
    assert sc[j + 1] - sc[j] > 1e-5
    return 0.5 * (sc[j] + sc[j + 1])


def _record_builds(monkeypatch, evaluation):
    """the byte capacity of every GraphedRawDetect evaluation builds, in order"""
    built, cls = [], evaluation.GraphedRawDetect

    def build(*args, **kw):
        det = cls(*args, **kw)
        built.append(det.max_bytes)
        return det

    monkeypatch.setattr(evaluation, 'GraphedRawDetect', build)
    return built


def _check_rebuild(built):
    """one graph for batch 1, rebuilt once, for batch 2, with at least twice the byte capacity"""
    print('GraphedRawDetect byte capacities: %s' % built)
    assert len(built) == 2 and built[1] >= 2 * built[0], built


@pytest.mark.gpu
def test_evaluate_with_raw_collater_equals_host_chain(monkeypatch):
    """evaluate(collater=RawCollater(pixel_scale=255), num_workers=2) on uint8 images == evaluate() on a dataset whose
    __getitem__ runs the host chain on the same images; batch 2 forces the byte-capacity rebuild, batch 3 is short.
    Ground truth: the model's own detections above a wide score gap, in original image coordinates"""
    from models import evaluation
    from models.pipeline import RawCollater
    S, n = 256, 10
    images = _eval_images(n, seed=61)
    m, K = _eval_model(0.3)
    host = _VOCSet(images, None, K, S, 255, raw=False)
    dets = []
    with torch.no_grad():
        for i in range(n):
            d = host[i]
            s, lab, box = m(d['img'].permute(2, 0, 1)[None].to(_dev()))
            dets.append((s.cpu().numpy(), lab.cpu().numpy(), box.cpu().numpy() / d['scale']))
    s_star = _gap(np.concatenate([d[0] for d in dets]))
    anns = [np.array([list(b) + [c] for s, c, b in zip(*d) if s > s_star] + [[1000, 1000, 1010, 1010, 7]], np.float64)
            for d in dets]
    host.annotations = anns
    want = evaluation.evaluate(host, m, batch_size=4)
    built = _record_builds(monkeypatch, evaluation)
    got = evaluation.evaluate(_VOCSet(images, anns, K, S, 255, raw=True), m, batch_size=4,
                              collater=RawCollater(S, pixel_scale=255), num_workers=2)
    _check_rebuild(built)
    print('VOC mAP: host chain %.6f, raw batches %.6f' % (want[0], got[0]))
    assert 0 < want[0] < 1
    assert abs(got[0] - want[0]) < 1e-6
    for c in range(K):
        assert got[1][c][1] == want[1][c][1] and abs(got[1][c][0] - want[1][c][0]) < 1e-6, c


class _CocoSet(_VOCSet):
    set_name = 'rawcase'

    def __init__(self, images, K, S, raw, inst, ids):
        super().__init__(images, None, K, S, None, raw)
        import coco_eval_oracle as CO
        self.coco, self.image_ids = CO.COCO(inst), ids

    def label_to_coco_label(self, label):
        return 2 * label + 1


@pytest.mark.gpu
def test_evaluate_coco_with_raw_collater_equals_host_chain(monkeypatch, tmp_path):
    """evaluate_coco(collater=RawCollater(), num_workers=2) against evaluate_coco() on the host chain's float images, with
    the byte-capacity rebuild and a short last batch.  The images are bit-identical, but two passes of the network
    differ in the last bits (the SE-mean fp32 atomics), and with many detections an NMS decision can follow that noise,
    so the stats are held to test_coco_eval's end-to-end bound of 1e-3."""
    from models import evaluation
    from models.pipeline import RawCollater
    monkeypatch.chdir(tmp_path)
    S, n = 256, 10
    images = _eval_images(n, seed=62, high=2)      # COCO's encoding is float32(u8): keep the network's input near 1
    m, K = _eval_model(0.3)
    ids = [int(v) for v in np.random.RandomState(4).permutation(np.arange(100, 100 + n))]
    inst = {'images': [{'id': i} for i in ids], 'categories': [{'id': 2 * k + 1} for k in range(K)], 'annotations': []}
    host = _CocoSet(images, K, S, False, inst, ids)
    res = []
    with torch.no_grad():
        for i in range(n):
            d = host[i]
            s, lab, box = m(d['img'].permute(2, 0, 1)[None].to(_dev()))
            for sc, c, b in zip(s.tolist(), lab.tolist(), (box / d['scale']).tolist()):
                res.append((ids[i], 2 * c + 1, sc, b))
    s_star = _gap(np.array([r[2] for r in res]))
    anns, per = [], {}
    for i, c, sc, (x1, y1, x2, y2) in res:                               # at most 20 per (image, category)
        per[i, c] = per.get((i, c), 0) + 1
        if sc > s_star and per[i, c] <= 20:
            anns.append({'id': len(anns) + 1, 'image_id': i, 'category_id': c, 'bbox': [x1, y1, x2 - x1, y2 - y1],
                         'area': (x2 - x1) * (y2 - y1), 'iscrowd': 0})
    for i in ids:                                                        # never matched: recall < 1
        anns.append({'id': len(anns) + 1, 'image_id': i, 'category_id': 15, 'bbox': [1000, 1000, 10, 10], 'area': 100,
                     'iscrowd': 0})
    inst['annotations'] = anns
    host = _CocoSet(images, K, S, False, inst, ids)
    want = evaluation.evaluate_coco(host, m, batch_size=4, max_records=1 << 20)
    m.eval()
    built = _record_builds(monkeypatch, evaluation)
    got = evaluation.evaluate_coco(_CocoSet(images, K, S, True, inst, ids), m, batch_size=4, collater=RawCollater(S),
                                   num_workers=2, max_records=1 << 20)
    _check_rebuild(built)
    print('COCO stats: host chain %s\n            raw batches %s' % (np.round(want, 6), np.round(got, 6)))
    assert want is not None and 0 < want[0] < 1
    assert np.abs(np.asarray(got) - np.asarray(want)).max() < 1e-3


@pytest.mark.gpu
def test_raw_graphs_capture_while_another_thread_pins_memory():
    """a DataLoader's pin thread allocates pinned memory while evaluate() / a training loop builds its raw graph; those
    allocations must not invalidate the capture.  A thread allocates fresh pinned blocks for the whole construction of
    a GraphedRawDetect and of a raw GraphedTrainStep; both build, and the detection replays"""
    import threading
    from models.graph_step import GraphedRawDetect, GraphedTrainStep
    from models.pipeline import RawCollater
    stop, held = threading.Event(), []

    def pin():
        while not stop.is_set() and len(held) < 2000:
            held.append(torch.empty((1 << 16) + 16 * len(held), dtype=torch.uint8, pin_memory=True))

    raw = RawCollater(128)(_samples(71, [(100, 120), (90, 60)], [2, 1]))
    m, _ = _eval_model(0.3)
    mt = _model(seed=72)
    t = threading.Thread(target=pin)
    t.start()
    try:
        det = GraphedRawDetect(m, raw)
        step = GraphedTrainStep(mt, raw, max_annotations=4, warmup=1)
    finally:
        stop.set()
        t.join()
    print('pinned blocks allocated during the captures: %d' % len(held))
    held.clear()
    out, scales = det(raw)
    torch.cuda.synchronize()
    assert out.count.shape == (2,) and np.array_equal(scales, raw.scales) and float(step(raw)) > 0
