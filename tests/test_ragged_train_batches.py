"""Training on the batches a DataLoader with collate_fn=collater yields: annotation tables whose width changes every batch,
images with more than 256 annotations, and a short last batch, all through one CUDA graph.

Three layers are checked.  The counted FocalLoss kernels (effdet_focal_loss_counted_fwd / _bwd) against the fp64
restatement of test_focal_loss_parity.py at any G and against the uncounted kernels where both run; the packing kernel
(effdet_pack_annots) against NumPy; and GraphedTrainStep(max_annotations=...) against the eager drop-in loop on the
same unpadded batches.  Every bound has a negative control that must exceed it."""
import collections
import os
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O
from test_focal_loss_parity import LOSS_RTOL, compare, rel, within
from test_graphed_train_loop import D0_MEDIAN, D0_WORST, _d0, _free_port, _rel
from test_host_trace import Recorder, traced  # noqa: F401  (traced is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
FAKE = 1 << 20                                               # aligned non-null "pointer"; never dereferenced


def _dev():
    return torch.device('cuda:0')


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument refusals of the new entry points, and the calls an eager step makes
# ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def _err(lib):
    return lib.effdet_last_error().decode()


@pytest.mark.parametrize('name', ['effdet_focal_loss_counted_fwd', 'effdet_focal_loss_counted_bwd'])
def test_counted_loss_refuses_bad_arguments_before_any_launch(lib, name):
    fn = getattr(lib, name)
    npt = 8 if name.endswith('fwd') else 10
    who = name[len('effdet_'):]

    def call(ptrs=None, B=2, A=100, K=20, G=300):
        return fn(*(ptrs or [FAKE] * npt), B, A, K, G, 0.25, 2.0, 0, None)

    for i in range(npt):                                     # every pointer, counts included
        ptrs = [FAKE] * npt
        ptrs[i] = None
        assert call(ptrs) == -1 and who in _err(lib) and 'null' in _err(lib), i
    for bad in (dict(B=0), dict(B=65536), dict(G=0), dict(G=-3), dict(G=(1 << 31) // 5 + 1), dict(A=0), dict(K=0)):
        assert call(**bad) == -1 and who in _err(lib), bad
    assert call(B=65536) == -1 and 'B=65536' in _err(lib)
    assert call(G=0) == -1 and 'G=0' in _err(lib)
    if not torch.cuda.is_available():                        # G far above 256 passes validation: only the device fails
        assert call(G=100000) < 0 and 'cuda' in _err(lib).lower() and who not in _err(lib)


def test_pack_refuses_batches_that_do_not_fit(lib):
    def call(B=3, G=7, Bcap=4, Gcap=8, ptrs=(FAKE, FAKE, FAKE)):
        a, o, c = ptrs
        return lib.effdet_pack_annots(a, B, G, o, c, Bcap, Gcap, 0, None)

    for i in range(3):
        ptrs = [FAKE] * 3
        ptrs[i] = None
        assert call(ptrs=ptrs) == -1 and 'pack_annots' in _err(lib) and 'null' in _err(lib), i
    assert call(B=5) == -1 and 'pack_annots' in _err(lib) and 'B=5' in _err(lib)
    assert call(G=9) == -1 and 'pack_annots' in _err(lib) and 'max_annotations=9 would be enough' in _err(lib)
    for bad in (dict(B=0), dict(G=0), dict(Bcap=0, B=1), dict(Gcap=0, G=1), dict(Bcap=65536)):
        assert call(**bad) == -1 and 'pack_annots' in _err(lib), bad
    if not torch.cuda.is_available():
        assert call(B=4, G=8) < 0 and 'pack_annots' not in _err(lib) and 'cuda' in _err(lib).lower()


def _ragged(counts, size, K, seed, G=None):
    """a collated annotation batch [B, G, 5]: image b has counts[b] boxes, -1 rows after them; G = max(counts, 1)"""
    g = torch.Generator().manual_seed(seed)
    G = G or max(max(counts), 1)
    ann = torch.full((len(counts), G, 5), -1.0)
    for b, n in enumerate(counts):
        if n:
            xy = torch.rand(n, 2, generator=g) * size * 0.8
            wh = 8 + torch.rand(n, 2, generator=g) * (size * 0.25 - 8)
            ann[b, :n, :2], ann[b, :n, 2:4] = xy, xy + wh
            ann[b, :n, 4] = torch.randint(0, K, (n,), generator=g).float()
    return ann


def test_eager_step_routes_wide_tables_to_the_counted_pair(traced):  # noqa: F811
    """an eager D0 step with G = 300 calls the counted pair with a [1 + B] counts buffer; with G <= 256 the step records
    exactly the uncounted calls, and both steps are otherwise the same call sequence"""
    rec, N = traced
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=2))
    m.train()
    m.is_training = True
    m.freeze_bn()
    images, _ = O.synthetic_batch(3, size=256, num_classes=20, seed=4)
    checked, recorder_check = [], rec.check

    def check(name, snap):                                   # buffer extents at call time, before any reuse
        recorder_check(name, snap)
        if name in ('effdet_focal_loss_counted_fwd', 'effdet_focal_loss_counted_bwd'):
            B, A, K, G = snap[-6:-2]
            rec.need(snap[0], B * A * K, 'cls'); rec.need(snap[1], B * A * 4, 'reg'); rec.need(snap[2], A * 4, 'anchors')
            rec.need(snap[3], B * G * 5, 'annots')
            rec.need(snap[4], 1 + B, 'counts')               # int32: one 4-byte element per entry
            checked.append((name, B, G))

    rec.check = check
    steps = {}
    for G in (256, 300, 8, 256):
        ann = _ragged([G, 5, 1], 256, 20, seed=G)
        for p in m.parameters():
            p.grad = None
        start = len(rec.calls)
        cl, rl = m([images, ann])
        (cl.mean() + rl.mean()).backward()
        steps[G] = rec.calls[start:]
    names = {G: [n for n, _ in calls] for G, calls in steps.items()}
    focal = {'effdet_focal_loss_fwd': 'effdet_focal_loss_counted_fwd', 'effdet_focal_loss_bwd': 'effdet_focal_loss_counted_bwd'}
    assert names[8] == names[256] and not set(focal.values()) & set(names[256])
    assert collections.Counter(names[256])['effdet_focal_loss_fwd'] == 1
    assert names[300] == [focal.get(n, n) for n in names[256]]
    assert checked == [('effdet_focal_loss_counted_fwd', 3, 300), ('effdet_focal_loss_counted_bwd', 3, 300)]
    for name, snap in steps[300]:
        assert len(snap) == len(N.SIGNATURES[name]) - 2, name
        if name in focal.values():
            assert (snap[-2], snap[-1]) == (0.25, 2.0)
    for name, snap in steps[256]:
        if name in focal:
            assert len(snap) == {'effdet_focal_loss_fwd': 13, 'effdet_focal_loss_bwd': 15}[name] and snap[-3] == 256


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level
# ------------------------------------------------------------------------------------------------------------------

def run_counted(cls, reg, anchors, annots, counts, alpha=0.25, gamma=2.0, gout=(1.5, 0.5)):
    """the counted pair, called the way FocalLossFn calls it; returns what test_focal_loss_parity.run_kernels returns"""
    from models import _native as N
    B, A, K = cls.shape
    G = annots.shape[1]
    dev = cls.device
    counts = torch.tensor(counts, dtype=torch.int32, device=dev)
    losses = torch.empty(2, device=dev)
    assign = torch.empty((B, A), dtype=torch.int32, device=dev)
    stats = torch.empty((B, 4), device=dev)
    N.call('effdet_focal_loss_counted_fwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors), N.f32(annots), counts.data_ptr(),
           N.f32(losses), assign.data_ptr(), N.f32(stats), B, A, K, G, float(alpha), float(gamma))
    g = torch.tensor(gout, dtype=torch.float32, device=dev)
    dcls, dreg = torch.full_like(cls, float('nan')), torch.full_like(reg, float('nan'))
    N.call('effdet_focal_loss_counted_bwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors), N.f32(annots), counts.data_ptr(),
           N.f32(g), assign.data_ptr(), N.f32(stats), N.f32(dcls), N.f32(dreg), B, A, K, G, float(alpha), float(gamma))
    torch.cuda.synchronize()
    st = stats.cpu().double()
    return dict(state=assign, npos=[int(v) for v in st[:, 0]], csum=st[:, 1].tolist(), rsum=st[:, 2].tolist(),
                loss=losses.cpu().double().tolist(), dcls=dcls, dreg=dreg)


def _wide_tables(anchors, B, G, H, W, K, seed):
    """[B, G, 5]: random boxes, a -1 row every 7th row, and at each chunk boundary that fits (rows 255/256 and 511/512)
    two copies of one anchor's box with different labels, so that anchor's first maximum is the earlier row"""
    rng = np.random.RandomState(seed)
    t = np.zeros((B, G, 5), np.float32)
    for b in range(B):
        x, y = rng.uniform(-8, W - 24, G), rng.uniform(-8, H - 24, G)
        w, h = rng.uniform(16, 96, G), rng.uniform(16, 96, G)
        t[b] = np.stack([x, y, x + w, y + h, rng.randint(K, size=G)], 1)
        t[b, 3::7] = -1.0
        pairs = [(r - 1, r) for r in (256, 512) if r < G] or [(G - 2, G - 1)]
        for i, (r0, r1) in enumerate(pairs):
            a = anchors[(7919 * (b + 1) + 104729 * i) % len(anchors)]
            t[b, r0, :4] = t[b, r1, :4] = a
            t[b, r0, 4], t[b, r1, 4] = i % K, (i + 1) % K
    return torch.from_numpy(t)


def _inputs(H, W, B, K, seed):
    d = _dev()
    anchors = torch.from_numpy(O.anchors_for(H, W)[0])
    g = torch.Generator(device=d).manual_seed(seed)
    A = anchors.shape[0]
    cls = torch.rand(B, A, K, generator=g, device=d) * 0.2
    reg = torch.randn(B, A, 4, generator=g, device=d) * 0.3
    return cls, reg, anchors


def _assign_last(anchors, ann):
    """assign_ref with the LAST maximum instead of the first: the negative control of the tie rule"""
    rows = torch.nonzero(ann[:, 4] != -1).flatten()
    iou = O.pairwise_iou(anchors, ann[rows, :4])
    m = iou.max(dim=1).values
    last = torch.where(iou == m[:, None], torch.arange(rows.numel(), device=iou.device)[None], -1).max(dim=1).values
    state = torch.where(torch.ge(m, 0.5), rows[last], -2)
    return torch.where(torch.lt(m, 0.4), -1, state).int()


@pytest.mark.gpu
@pytest.mark.parametrize('G', [256, 257, 1000, 3000])
def test_counted_kernels_match_restatement_at_any_width(G):
    H = W = 512
    B, K = 2, 20
    cls, reg, anchors = _inputs(H, W, B, K, seed=G)
    annots = _wide_tables(anchors.numpy(), B, G, H, W, K, seed=G).to(_dev())
    anchors = anchors.to(_dev())
    out = run_counted(cls, reg, anchors, annots, [B] + [G] * B)
    m = compare(out, cls, reg, anchors, annots)
    flips = sum(int((_assign_last(anchors, annots[b]) != out['state'][b]).sum()) for b in range(B))
    straddle = [int(((out['state'][b] == 255) | (out['state'][b] == 511)).sum()) for b in range(B)]
    print('G=%d: %s, positives %s, anchors on a boundary tie %s, last-maximum control flips %d states'
          % (G, m, out['npos'], straddle, flips))
    assert not within(m), m
    if G > 256:
        assert min(straddle) > 0                             # the tie across the chunk boundary was exercised
    assert flips > 0


@pytest.mark.gpu
@pytest.mark.parametrize('case', [('d0', 512, 512, 32, 80, 8), ('k20', 512, 512, 2, 20, 24), ('full', 384, 640, 3, 3, 256)])
def test_counted_equals_uncounted_where_both_run(case):
    """counts = (B, G, ..., G) at G <= 256: states, positive counts, dcls and dreg bit-equal to the uncounted pair;
    control: the same call with n_img = B - 1 changes the gradient scale of every image"""
    from test_focal_loss_parity import run_kernels
    name, H, W, B, K, G = case
    cls, reg, anchors = _inputs(H, W, B, K, seed=B * K)
    _, syn = O.synthetic_batch(B, size=min(H, W), G=G, num_classes=K, seed=1)
    anchors, annots = anchors.to(_dev()), syn.to(_dev())
    old = run_kernels(cls, reg, anchors, annots)
    new = run_counted(cls, reg, anchors, annots, [B] + [G] * B)
    assert torch.equal(old['state'], new['state']) and old['npos'] == new['npos']
    assert torch.equal(old['dcls'], new['dcls']) and torch.equal(old['dreg'], new['dreg'])
    err = max(rel(a, b) for a, b in zip(new['loss'], old['loss']))
    assert err <= LOSS_RTOL, err
    ctrl = run_counted(cls, reg, anchors, annots, [B - 1] + [G] * B)
    assert not torch.equal(old['dcls'][0], ctrl['dcls'][0])
    print('%s: loss rel diff %.2e, positives %s' % (name, err, new['npos'][:4]))


@pytest.mark.gpu
def test_padding_images_and_rows_past_the_count_are_never_read():
    """n_img = 3 of B = 5: the padding images' cls / reg are NaN and every image has valid-looking boxes past its count.
    Images b < n_img equal a run on those images alone with the rows truncated, bit for bit; padding dcls / dreg are
    exactly 0; the losses are the mean over n_img.  Control: the mean over B."""
    from test_focal_loss_parity import run_kernels
    H = W = 512
    B, K, n = 5, 20, 3
    cls, reg, anchors = _inputs(H, W, B, K, seed=5)
    anchors = anchors.to(_dev())
    rows = [7, 0, 40]
    full = _ragged([60] * B, H, K, seed=9).to(_dev())           # every row valid-looking
    cls[n:], reg[n:] = float('nan'), float('nan')
    out = run_counted(cls, reg, anchors, full, [n] + rows + [60, 60])
    alone = full[:n, :max(rows)].clone()
    for b, c in enumerate(rows):
        alone[b, c:] = -1.0
    ref = run_kernels(cls[:n].contiguous(), reg[:n].contiguous(), anchors, alone.contiguous())
    assert torch.equal(out['state'][:n], ref['state']) and out['npos'][:n] == ref['npos']
    assert torch.equal(out['dcls'][:n], ref['dcls']) and torch.equal(out['dreg'][:n], ref['dreg'])
    assert bool((out['state'][n:] == -3).all()) and out['npos'][n:] == [0, 0]
    assert out['csum'][n:] == [0.0, 0.0] and out['rsum'][n:] == [0.0, 0.0]
    pad_c, pad_r = out['dcls'][n:], out['dreg'][n:]
    assert bool((pad_c == 0).all()) and bool((pad_r == 0).all())
    assert not bool(torch.signbit(pad_c).any()) and not bool(torch.signbit(pad_r).any())   # +0.0, written, not NaN
    err = max(rel(a, b) for a, b in zip(out['loss'], ref['loss']))
    ctrl = max(rel(a * n / B, b) for a, b in zip(out['loss'], ref['loss']))
    print('n_img %d of %d: loss rel diff %.2e, mean-over-B control %.2e' % (n, B, err, ctrl))
    assert err <= LOSS_RTOL and ctrl > LOSS_RTOL


def _pack_ref(ann, Bcap, Gcap):
    B = ann.shape[0]
    out = np.full((Bcap, Gcap, 5), -1.0, np.float32)
    counts = np.zeros(1 + Bcap, np.int32)
    counts[0] = B
    for b in range(B):
        keep = ann[b][ann[b, :, 4] != -1]
        out[b, :len(keep)] = keep
        counts[1 + b] = len(keep)
    return out, counts


@pytest.mark.gpu
@pytest.mark.parametrize('B,G,Bcap,Gcap,empty', [(3, 7, 5, 9, (1,)), (4, 1, 4, 4, (0, 1, 2, 3)), (2, 600, 4, 600, ()),
                                                 (5, 256, 8, 256, (4,)), (32, 40, 32, 256, ())])
def test_pack_matches_numpy(B, G, Bcap, Gcap, empty):
    """ragged batches into a static table: B < Bcap, images without boxes, the collater's single -1 row when no image
    has boxes, G = Gcap; -1 rows interleaved to check the compaction is stable.  Control: a reversed order differs."""
    from models import _ops
    rng = np.random.RandomState(B * 1000 + G)
    ann = _ragged([int(c) for c in rng.randint(1, G + 1, size=B)], 512, 20, seed=G, G=G).numpy()
    ann[:, 1::3, 4] = -1                                     # interleaved -1 rows (labels only: the boxes stay)
    for b in empty:
        ann[b] = -1
    out = torch.full((Bcap, Gcap, 5), float('nan'), device=_dev())
    counts = torch.full((1 + Bcap,), -7, dtype=torch.int32, device=_dev())
    _ops.pack_annotations(torch.from_numpy(ann).to(_dev()), out, counts)
    want, want_c = _pack_ref(ann, Bcap, Gcap)
    got, got_c = out.cpu().numpy(), counts.cpu().numpy()
    assert np.array_equal(got_c, want_c), (got_c, want_c)
    assert np.array_equal(got, want)
    b = int(np.argmax(want_c[1:]))
    if want_c[1 + b] > 1:
        rev = want.copy()
        rev[b, :want_c[1 + b]] = rev[b, :want_c[1 + b]][::-1]
        assert not np.array_equal(got, rev)


# ------------------------------------------------------------------------------------------------------------------
# GPU, model level: D0 W64 D2 (model.eval(); is_training = True), capacity-mode graphed loop against the eager loop
# ------------------------------------------------------------------------------------------------------------------

# micro-batches as collater makes them: per-image box counts, each batch padded to its own largest count
EPOCH = [[300, 12, 5, 1], [1, 1, 1, 1], [40, 3, 17, 8], [0, 0, 0, 0], [9, 0, 22, 4], [7, 15, 2]]


def _epoch(size=256, Bcap=4):
    batches = []
    for i, counts in enumerate(EPOCH):
        images = torch.randn(len(counts), 3, size, size, generator=torch.Generator().manual_seed(60 + i))
        batches.append((images.to(_dev()), _ragged(counts, size, 20, seed=70 + i).to(_dev())))
    return batches


def _eager(m, opt, batches, k, tail_scale=1.0):
    """the drop-in loop (train.py:107-118) on the unpadded batches; tail_scale multiplies the last batch's loss"""
    losses = []
    opt.zero_grad()
    for idx, (images, annotations) in enumerate(batches):
        cl, rl = m([images, annotations])
        loss = cl.mean() + rl.mean()
        if idx == len(batches) - 1:
            loss = loss * tail_scale
        if bool(loss == 0):
            losses.append(0.0)
            continue
        loss.backward()
        if (idx + 1) % k == 0:
            opt.step()
            opt.zero_grad()
        losses.append(loss.item())
    return losses


@pytest.mark.gpu
def test_dataloader_shaped_epoch_matches_eager_drop_in():
    """Bcap = 4, Gcap = 512, k = 2: batch widths 1..300, a batch without annotations, a last batch of 3 images.  Each
    micro-step loss within 1e-3 of the eager loop's, the parameter updates within test_graphed_train_loop's D0 bounds,
    equal step counts.  Controls: the tail loss averaged over Bcap, and the graphed loop without the tail."""
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=43)
    batches = _epoch()
    k = 2

    def eager(tail_scale):
        m = _d0(sd)
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        losses = _eager(m, opt, batches, k, tail_scale)
        torch.cuda.synchronize()
        steps = {int(st['step']) for st in opt.state_dict()['state'].values()}
        return {n: p.detach() - p0[n] for n, p in m.named_parameters()}, losses, steps

    upd_e, loss_e, steps_e = eager(1.0)
    upd_b, loss_b, _ = eager(3 / 4)                          # the tail's loss averaged over Bcap = 4 images, not 3
    m = _d0(sd)
    p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    step = GraphedTrainStep(m, batches[0][0], batches[0][1], optimizer=opt, max_annotations=512)
    opt.zero_grad()
    loss_g = []
    for idx, (images, ann) in enumerate(batches):
        loss_g.append(float(step(images, ann, update=(idx + 1) % k == 0)))
        if idx == len(batches) - 2:                          # the graphed loop without the tail: the update at idx 5
            upd_d = {n: p.detach() - p0[n] for n, p in m.named_parameters()}   # has not run yet
    upd_g = {n: p.detach() - p0[n] for n, p in m.named_parameters()}
    steps_g = {int(st['step']) for st in opt.state_dict()['state'].values()}

    def errs(upd):
        e = sorted(_rel(upd[n], upd_e[n]) for n in upd_e if float(upd_e[n].abs().max()) > 0)
        return e[len(e) // 2], e[-1], len(e)

    def loss_err(ls):
        return max(abs(a - b) / abs(b) for a, b in zip(ls, loss_e) if b != 0)

    med, worst_, n = errs(upd_g)
    print('capacity-mode epoch: losses %s vs eager %s; %d updated tensors, update rel err median %.2e worst %.2e; '
          'loss rel err %.2e' % (['%.5f' % v for v in loss_g], ['%.5f' % v for v in loss_e], n, med, worst_,
                                 loss_err(loss_g)))
    print('controls: tail over Bcap loss err %.2e, update median %.2e; without the tail update median %.2e worst %.2e'
          % (loss_err(loss_b), errs(upd_b)[0], *errs(upd_d)[:2]))
    assert loss_g[3] == 0.0 and loss_e[3] == 0.0
    assert loss_err(loss_g) < 1e-3
    assert n > 250 and med < D0_MEDIAN and worst_ < D0_WORST
    assert steps_g == steps_e == {2}                         # boundaries 1 and 5; 3 has no annotations
    assert loss_err(loss_b) > 1e-3 and errs(upd_b)[0] > D0_MEDIAN
    assert errs(upd_d)[0] > D0_MEDIAN


@pytest.mark.gpu
def test_capacity_mode_at_the_bench_geometry_matches_the_default_step():
    """D0 512^2, Bcap = 32, Gcap = 256: one replay on a full ragged batch (VOC-like counts) against the default
    GraphedTrainStep on the same batch padded to its own G"""
    from models.graph_step import GraphedTrainStep
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    m = _d0(O.init_state_dict(cfg, seed=44))
    rng = np.random.RandomState(45)
    counts = [int(c) for c in np.minimum(rng.geometric(0.25, size=32), 40)]
    images = torch.randn(32, 3, 512, 512, generator=torch.Generator().manual_seed(46)).to(_dev())
    ann = _ragged(counts, 512, 20, seed=47).to(_dev())
    step = GraphedTrainStep(m, images, ann, max_annotations=256)
    cap = float(step(images, ann))
    del step
    torch.cuda.empty_cache()
    step = GraphedTrainStep(m, images, ann)
    ref = float(step(images, ann))
    print('bench geometry, G = %d: capacity mode %.7f, default step %.7f, rel diff %.2e'
          % (ann.shape[1], cap, ref, abs(cap - ref) / abs(ref)))
    assert abs(cap - ref) <= 1e-5 * abs(ref)


@pytest.mark.gpu
def test_batches_that_do_not_fit_are_refused_without_side_effects():
    from models import _native as N
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    m = _d0(O.init_state_dict(cfg, seed=48))
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    images = torch.randn(2, 3, 128, 128, generator=torch.Generator().manual_seed(49)).to(_dev())
    ann = _ragged([3, 5], 128, 20, seed=50).to(_dev())
    with pytest.raises(N.EffdetNativeError, match='max_annotations=4 or more'):
        GraphedTrainStep(m, images, _ragged([4, 1], 128, 20, seed=1).to(_dev()), optimizer=opt, max_annotations=3)
    with pytest.raises(N.EffdetNativeError, match='max_annotations must be an integer'):
        GraphedTrainStep(m, images, ann, optimizer=opt, max_annotations=0)
    step = GraphedTrainStep(m, images, ann, optimizer=opt, max_annotations=8)
    step(images, ann, update=True)
    torch.cuda.synchronize()
    G = opt._graph

    def state():
        return [t.clone() for t in [step.static_images, step.static_annots, step.static_counts, G['step'], G['lr'],
                                    G['update']] + [p.detach() for p in m.parameters()]
                + [p.grad for p in m.parameters() if p.grad is not None]
                + [v for st in opt.state.values() for v in st.values() if torch.is_tensor(v)]]

    before = state()
    launches = N.launch_count()
    refusals = [(torch.randn(3, 3, 128, 128, device=_dev()), _ragged([1, 1, 1], 128, 20, seed=2).to(_dev()), 'capacity of 2'),
                (images[:1], _ragged([9], 128, 20, seed=3).to(_dev()), 'max_annotations=9 or more'),
                (torch.randn(2, 3, 160, 128, device=_dev()), ann, 'captured for images'),
                (images, ann[:1], 'annotations must be')]
    for imgs, a, msg in refusals:
        with pytest.raises(N.EffdetNativeError, match=msg):
            step(imgs, a.cpu(), update=False)
    torch.cuda.synchronize()
    assert N.launch_count() == launches and G['update_host'] == 1
    for a, b in zip(before, state()):
        assert torch.equal(a, b)
    loss = step(images[:1], ann[:1].cpu(), update=True)           # a host batch of one still runs after the refusals
    assert float(loss) > 0 and int(step.static_counts[0]) == 1 and bool((step.static_images[1:] == 0).all())


# ------------------------------------------------------------------------------------------------------------------
# GPU, 2 ranks: capacity mode over the DDP wrapper with a short, ragged last batch
# ------------------------------------------------------------------------------------------------------------------

def _ddp_worker(rank, world, port, out):
    os.environ['TORCH_NCCL_ASYNC_ERROR_HANDLING'] = '0'
    os.environ['NCCL_ASYNC_ERROR_HANDLING'] = '0'
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    for p in (os.path.join(os.path.dirname(HERE), 'oracle'), os.path.join(os.path.dirname(HERE), 'efficientdet.pytorch_b200')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    from models import EfficientDet
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=3)
    plan = [([4, 30], [2, 11]), ([1, 7], [19, 3]), ([5], [2])]          # per rank: box counts; the last batch is short
    batches = []
    for i, per_rank in enumerate(plan):
        counts = per_rank[rank]
        images = torch.randn(len(counts), 3, 256, 256, generator=torch.Generator().manual_seed(90 + 10 * i + rank))
        batches.append((images.to(dev), _ragged(counts, 256, 20, seed=95 + 10 * i + rank).to(dev)))
    res = {}
    for mode in ('graph', 'eager'):
        m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
        m.load_state_dict(sd)
        m = m.to(dev)
        m.eval()
        m.is_training = True
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            net = torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], find_unused_parameters=True,
                                                            static_graph=True, gradient_as_bucket_view=True,
                                                            broadcast_buffers=False)
        torch.cuda.current_stream(dev).wait_stream(side)
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        if mode == 'graph':
            step = GraphedTrainStep(net, batches[0][0], batches[0][1], optimizer=opt, max_annotations=64)
            for images, ann in batches:
                step(images, ann)
        else:
            with torch.cuda.stream(side):
                for images, ann in batches:
                    opt.zero_grad()
                    cl, rl = net([images, ann])
                    (cl.mean() + rl.mean()).backward()
                    opt.step()
        torch.cuda.synchronize()
        res[mode] = {n: (p.detach() - p0[n]).cpu() for n, p in m.named_parameters()}
        res[mode + '_step'] = int(next(iter(opt.state_dict()['state'].values()))['step'])
    torch.save(res, os.path.join(out, 'r%d.pt' % rank))
    torch.cuda.synchronize()
    dist.barrier(device_ids=[rank])
    os._exit(0)                                                 # (NCCL teardown after a captured collective hangs)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_capacity_mode_with_a_short_ragged_last_batch(tmp_path):
    """the two ranks' short last batches weigh in DDP's gradient average as they do in eager DDP: each rank's loss is
    the mean over its real images"""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_ddp_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp_path, 'r%d.pt' % r)) for r in (0, 1))
    assert r0['graph_step'] == r0['eager_step'] == 3
    errs = []
    for n, ref in r0['eager'].items():
        assert torch.equal(r0['graph'][n], r1['graph'][n]), 'ranks disagree on ' + n
        if float(ref.abs().max()) > 0:
            errs.append(_rel(r0['graph'][n], ref))
    errs.sort()
    print('DDP capacity mode vs eager: update rel err median %.2e worst %.2e' % (errs[len(errs) // 2], errs[-1]))
    assert errs[len(errs) // 2] < D0_MEDIAN and errs[-1] < D0_WORST
