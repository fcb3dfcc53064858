"""FocalLoss kernels (csrc/loss.cu) element by element against the reference and an fp64 restatement.

The loss is the only kernel on the training path whose output hangs on discrete fp32 decisions: each anchor's first
maximum IoU over the annotations, compared with 0.4 and 0.5, makes it background, ignored or positive and picks its
label and box.  A loss value cannot see one such decision go wrong (one background anchor among ~47,000 moves an
image's sum by ~2e-5), so the assignment is compared bit for bit and the gradients per element:

- states and positive counts: bit-equal;
- per-image sums and the two losses: LOSS_RTOL relative (fp32 atomics over up to 15.7 M terms per image);
- dcls: every element within DCLS_RTOL relative, and exactly 0.0 wherever the reference is 0 (ignored anchors, images
  without annotations, clamped probabilities);
- dreg: every element within DREG_RTOL * |ref| + 9 * gs * DREG_ULPS * ulp(t), gs the smooth-L1 gradient scale (the
  kernel's logf and the host's log may differ by an ulp in the target t), and exactly zero off the positives.

focal_ref() is the reference restated in fp64, except where the reference rounds in fp32 in a way fp64 cannot stand
in for: the IoU and the threshold tests (they decide the assignment), the clamped probability pc and 1 - pc (the
reference takes log(1 - pc) of the fp32 difference, which alone moves the gradient by ~2e-4 relative at p ~ 1e-4), and
the regression target t.  tests/golden/focal_loss.npz pins it to the reference's own loss code
(tests/golden/make_focal_golden.py).  Each comparison has a negative control: a reference corrupted by one flipped
state, one swapped label or a wrong positive count must exceed that comparison's bound."""
import math
import os
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import make_focal_golden as MG  # noqa: E402

LOSS_RTOL = 5e-5
DCLS_RTOL = 1e-5
DREG_RTOL = 1e-5
DREG_ULPS = 4


@pytest.fixture(scope='module')
def golden():
    return np.load(os.path.join(HERE, 'golden', 'focal_loss.npz'))


# ------------------------------------------------------------------------------------------------
# fp64 restatement of models/losses.py:32-152
# ------------------------------------------------------------------------------------------------

def assign_ref(anchors, ann):
    """(state [A] int32, iou_max [A] fp32) of one image.  state in the kernel's encoding: the unfiltered row of a
    positive anchor's first maximum, -1 background (IoU < 0.4), -2 ignored, -3 no annotation (losses.py:52, 63-76)"""
    A = anchors.shape[0]
    rows = torch.nonzero(ann[:, 4] != -1).flatten()
    if rows.numel() == 0:
        return (torch.full((A,), -3, dtype=torch.int32, device=anchors.device),
                torch.zeros(A, device=anchors.device))
    iou = O.pairwise_iou(anchors, ann[rows, :4])
    m = iou.max(dim=1).values
    n = rows.numel()
    first = torch.where(iou == m[:, None], torch.arange(n, device=iou.device)[None], n).min(dim=1).values
    state = torch.where(torch.ge(m, 0.5), rows[first], -2)
    state = torch.where(torch.lt(m, 0.4), -1, state)
    return state.int(), m


def labels_of(ann, state):
    """the class each anchor is trained toward: its annotation's label (.long(), losses.py:84), -1 if not positive"""
    return torch.where(state >= 0, ann[state.clamp(min=0).long(), 4].long(), -1)


def image_ref(cls, reg, anchors, ann, state, label, alpha, gamma):
    """one image's focal sum and smooth-L1 sum (fp64) and their derivatives w.r.t. cls [A,K] and reg [A,4] (fp64),
    and the fp32 regression targets t [A,4] (zero off the positives)"""
    A, K = cls.shape
    dev = cls.device
    dc = torch.zeros(A, K, dtype=torch.float64, device=dev)
    dr = torch.zeros(A, 4, dtype=torch.float64, device=dev)
    t32 = torch.zeros(A, 4, device=dev)
    live = state >= -1                                          # ignored anchors and images without boxes: no loss
    if not bool(live.any()):
        return 0.0, 0.0, dc, dr, t32
    pc32 = torch.clamp(cls, 1e-4, 1.0 - 1e-4)
    pc, q = pc32.double(), (1.0 - pc32).double()                # 1 - pc rounded in fp32, as the reference does
    tgt = torch.arange(K, device=dev)[None] == label[:, None]
    lp, lq = torch.log(pc), torch.log(q)
    loss = torch.where(tgt, alpha * q ** gamma * -lp, (1 - alpha) * pc ** gamma * -lq)
    d = torch.where(tgt, alpha * (gamma * q ** (gamma - 1) * lp - q ** gamma / pc),
                    (1 - alpha) * (-gamma * pc ** (gamma - 1) * lq + pc ** gamma / q))
    inside = (cls >= 1e-4) & (cls <= 1.0 - 1e-4)                # the clamp's backward, inclusive at both bounds
    csum = float(torch.where(live[:, None], loss, 0.0).sum())
    dc = torch.where(live[:, None] & inside, d, 0.0)
    rsum = 0.0
    pos = torch.nonzero(state >= 0).flatten()
    if pos.numel():
        g, a = ann[state[pos].long(), :4], anchors[pos]
        aw, ah = a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]
        acx, acy = a[:, 0] + 0.5 * aw, a[:, 1] + 0.5 * ah
        gw, gh = g[:, 2] - g[:, 0], g[:, 3] - g[:, 1]
        gcx, gcy = g[:, 0] + 0.5 * gw, g[:, 1] + 0.5 * gh
        gw, gh = torch.clamp(gw, min=1), torch.clamp(gh, min=1)
        t = torch.stack(((gcx - acx) / aw, (gcy - acy) / ah, torch.log(gw / aw), torch.log(gh / ah)), 1)
        t = t / torch.tensor([[0.1, 0.1, 0.2, 0.2]], device=dev)
        r = reg[pos]
        quad = torch.le(torch.abs(t - r), 1.0 / 9.0)           # the reference's fp32 branch test
        diff = r.double() - t.double()
        rsum = float(torch.where(quad, 4.5 * diff ** 2, diff.abs() - 0.5 / 9.0).sum())
        dr[pos] = torch.where(quad, 9.0 * diff, torch.sign(diff))
        t32[pos] = t
    return csum, rsum, dc, dr, t32


def grad_scales(B, npos, gout):
    """d loss / d (per-image sum): gout[0] / (B max(npos, 1)) for the focal sum, gout[1] / (4 B npos) for smooth-L1"""
    return gout[0] / (B * max(npos, 1)), (gout[1] / (4 * B * npos) if npos else 0.0)


def losses_ref(csum, rsum, npos):
    B = len(csum)
    return (sum(c / max(n, 1) for c, n in zip(csum, npos)) / B,
            sum(r / (4 * n) if n else 0.0 for r, n in zip(rsum, npos)) / B)


def focal_ref(cls, reg, anchors, annots, alpha=0.25, gamma=2.0, gout=(1.0, 1.0)):
    """the reference's FocalLoss forward and backward for upstream gradient gout: states [B,A], positive counts [B],
    per-image sums, the two losses and the closed-form dcls [B,A,K], dreg [B,A,4] (fp64)"""
    B = cls.shape[0]
    out = dict(state=[], npos=[], csum=[], rsum=[], dcls=[], dreg=[])
    for b in range(B):
        state, _ = assign_ref(anchors, annots[b])
        npos = int((state >= 0).sum())
        c, r, dc, dr, _ = image_ref(cls[b], reg[b], anchors, annots[b], state, labels_of(annots[b], state), alpha, gamma)
        gc, gr = grad_scales(B, npos, gout)
        for k, v in (('state', state), ('npos', npos), ('csum', c), ('rsum', r), ('dcls', gc * dc), ('dreg', gr * dr)):
            out[k].append(v)
    out['loss'] = losses_ref(out['csum'], out['rsum'], out['npos'])
    out['state'], out['dcls'], out['dreg'] = (torch.stack(out[k]) for k in ('state', 'dcls', 'dreg'))
    return out


# ------------------------------------------------------------------------------------------------
# comparisons
# ------------------------------------------------------------------------------------------------

def excess(k, r, bound):
    """largest |k - r| / bound over the elements; where the bound is zero the element must be exact, and a NaN
    anywhere is an infinite excess"""
    d = (k.double() - r).abs()
    over = torch.where(bound > 0, d / bound.clamp(min=1e-300), torch.where(d > 0, float('inf'), 0.0))
    over = torch.where(torch.isnan(d), float('inf'), over)
    return float(over.max()) if over.numel() else 0.0


def rel(k, r):
    """|k - r| / |r|; exact where r is 0, infinite where either is not finite"""
    k, r = float(k), float(r)
    if not (math.isfinite(k) and math.isfinite(r)):
        return float('inf')
    return abs(k - r) / abs(r) if r != 0 else (0.0 if k == 0 else float('inf'))


def worst(*errors):
    """the largest of the errors; NaN counts as the largest"""
    return float('inf') if any(e != e for e in errors) else max(errors)


def dreg_bound(r, t32, gr, ulps=DREG_ULPS):
    ulp = (torch.nextafter(t32.abs(), torch.tensor(float('inf'), device=t32.device)) - t32.abs()).double()
    return DREG_RTOL * r.abs() + 9 * abs(gr) * ulps * ulp * (t32 != 0)


def grad_excess(kc, kr, dc, dr, t32, gc, gr):
    rc, rr = gc * dc, gr * dr
    return excess(kc, rc, DCLS_RTOL * rc.abs()), excess(kr, rr, dreg_bound(rr, t32, gr))


def corrupted(kind, cls, state, label, npos):
    """the reference's state, labels and positive count with one fault"""
    state, label = state.clone(), label.clone()
    pos = torch.nonzero(state >= 0).flatten()
    if kind == 'state':                      # the positive anchor with the largest target term becomes ignored
        a = pos[torch.argmin(cls[pos, label[pos]])]
        state[a], label[a], npos = -2, -1, npos - 1
    elif kind == 'label':                    # a positive whose old and new target entries both have a gradient
        K = cls.shape[1]
        ok = [a for a in pos.tolist() if all(1e-4 <= float(cls[a, k]) <= 0.9999 for k in (label[a], (label[a] + 1) % K))]
        label[ok[0]] = (label[ok[0]] + 1) % K
    elif kind == 'npos':
        npos += 1
    return state, label, npos


def compare(out, cls, reg, anchors, annots, alpha=0.25, gamma=2.0, gout=(1.5, 0.5), fault=None):
    """worst error of each comparison between the kernels' outputs and the restatement, computed one image at a time
    on the inputs' device; fault corrupts the reference of image 0.  Without 'state' in out (a run through the
    module, which keeps its workspaces) only the losses and gradients are compared."""
    B = cls.shape[0]
    ws = 'state' in out
    m = dict(state=0, npos=0, csum=0.0, rsum=0.0, loss=0.0, dcls=0.0, dreg=0.0)
    csum, rsum, nposs = [], [], []
    for b in range(B):
        state, _ = assign_ref(anchors, annots[b])
        label, npos = labels_of(annots[b], state), int((state >= 0).sum())
        if fault and b == 0:
            state, label, npos = corrupted(fault, cls[b], state, label, npos)
        c, r, dc, dr, t32 = image_ref(cls[b], reg[b], anchors, annots[b], state, label, alpha, gamma)
        gc, gr = grad_scales(B, npos, gout)
        if ws:
            m['state'] += int((out['state'][b] != state).sum())
            m['npos'] += int(out['npos'][b] != npos)
            m['csum'] = worst(m['csum'], rel(out['csum'][b], c))
            m['rsum'] = worst(m['rsum'], rel(out['rsum'][b], r))
        ec, er = grad_excess(out['dcls'][b], out['dreg'][b], dc, dr, t32, gc, gr)
        m['dcls'], m['dreg'] = worst(m['dcls'], ec), worst(m['dreg'], er)
        csum.append(c), rsum.append(r), nposs.append(npos)
    lc, lr = losses_ref(csum, rsum, nposs)
    m['loss'] = worst(rel(out['loss'][0], lc), rel(out['loss'][1], lr))
    return m


def within(m):
    """the comparisons that fail their bound (dcls and dreg are reported as error / bound)"""
    bad = [k for k in ('state', 'npos') if m[k]]
    bad += [k for k in ('csum', 'rsum', 'loss') if not m[k] <= LOSS_RTOL]
    return bad + [k for k in ('dcls', 'dreg') if not m[k] <= 1.0]


# ------------------------------------------------------------------------------------------------
# CPU: the restatement against the reference's fixture, the closed form against autograd, the G bound
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', list(MG.BATCHES))
def test_restatement_matches_reference_fixture(golden, name):
    cls, reg, anchors, annots, _ = MG.make_batch(name)
    p = name + '/'
    assert np.array_equal(annots.numpy(), golden[p + 'annots'])
    gout = tuple(golden['gout'].tolist())
    ref = focal_ref(cls, reg, anchors, annots, gout=gout)
    assert np.array_equal(ref['state'].numpy(), golden[p + 'state'])
    assert ref['npos'] == golden[p + 'npos'].tolist()
    B = cls.shape[0]
    m = dict(loss=worst(*(rel(float(golden[p + 'losses'][i]), ref['loss'][i]) for i in range(2))), dcls=0.0, dreg=0.0)
    for b in range(B):
        state = ref['state'][b]
        c, r, dc, dr, t32 = image_ref(cls[b], reg[b], anchors, annots[b], state, labels_of(annots[b], state), 0.25, 2.0)
        gc, gr = grad_scales(B, ref['npos'][b], gout)
        ec, er = grad_excess(torch.from_numpy(golden[p + 'dcls'][b]), torch.from_numpy(golden[p + 'dreg'][b]),
                             dc, dr, t32, gc, gr)
        m['dcls'], m['dreg'] = worst(m['dcls'], ec), worst(m['dreg'], er)
    print('%s restatement vs reference: %s' % (name, m))
    assert m['loss'] <= LOSS_RTOL and m['dcls'] <= 1.0 and m['dreg'] <= 1.0, m


def test_fixture_holds_every_crafted_case(golden):
    """the crafted cases of make_focal_golden.py are in the fixture, with the reference's decision on each"""
    kinds, seen = [], set()
    H, W = MG.SIZE
    for name in MG.BATCHES:
        p = name + '/'
        cls, reg, anchors, annots, crafted = MG.make_batch(name)
        state, ann, npos = golden[p + 'state'], golden[p + 'annots'], golden[p + 'npos']
        assert [c[2] for c in crafted] == golden[p + 'crafted_kind'].tolist()
        for (b, a, kind, want), got in zip(crafted, golden[p + 'crafted_iou']):
            assert got == want, (name, kind, got, want)
            s = state[b, a]
            if kind.startswith('iou'):                         # the threshold decision at and next to 0.4 and 0.5
                assert (s >= 0) == (want >= np.float32(0.5)) and (s == -1) == (want < np.float32(0.4)), (kind, s)
            else:                                              # ties: the first of two rows with different labels
                iou = O.pairwise_iou(anchors[a:a + 1], torch.from_numpy(ann[b, :, :4]))[0].numpy()
                rows = np.nonzero((iou == want) & (ann[b, :, 4] != -1))[0]
                assert len(rows) == 2 and ann[b, rows[0], 4] != ann[b, rows[1], 4] and s == rows[0], (kind, rows, s)
            kinds.append(kind)
        real = ann[:, :, 4] != -1
        w, h = ann[..., 2] - ann[..., 0], ann[..., 3] - ann[..., 1]
        for b in range(len(ann)):
            last = np.nonzero(real[b])[0][-1] if real[b].any() else -1
            seen |= {'padding between rows'} if not real[b, :last].all() else set()
            seen |= {'padding only'} if not real[b].any() else set()
            seen |= {'no positive'} if real[b].any() and npos[b] == 0 else set()
        seen |= {'zero width'} if (real & (w == 0)).any() else set()
        seen |= {'sub-pixel'} if (real & (w > 0) & (w < 1) & (h < 1)).any() else set()
        seen |= {'outside'} if (real & ((ann[..., 2] > W) | (ann[..., 3] > H) | (ann[..., 0] < 0))).any() else set()
        # clamp-boundary probabilities on target entries of positive anchors and on other contributing entries
        bb, aa = np.nonzero(state >= 0)
        target_p = cls.numpy()[bb, aa, ann[bb, state[bb, aa], 4].astype(np.int64)]
        live = cls.numpy()[state >= -1]
        for v in MG.SPECIAL_P:
            assert (target_p == v).any() and (live == v).any(), (name, v)
    assert sorted(kinds) == sorted(['iou0.5+0', 'iou0.4+0', 'iou0.5-2', 'iou0.5-1', 'iou0.5+1', 'iou0.5+2', 'iou0.4-2',
                                    'iou0.4-1', 'iou0.4+1', 'iou0.4+2', 'tie_duplicate', 'tie_mirror'] * 2)
    assert seen == {'padding between rows', 'padding only', 'no positive', 'zero width', 'sub-pixel', 'outside'}


def _sides(cls, reg, anchors, annots):
    """|t - r| at the positives, from the restatement's fp32 targets"""
    d = []
    for b in range(cls.shape[0]):
        state, _ = assign_ref(anchors, annots[b])
        _, _, _, _, t32 = image_ref(cls[b], reg[b], anchors, annots[b], state, labels_of(annots[b], state), 0.25, 2.0)
        d.append((t32[state >= 0] - reg[b][state >= 0]).abs().flatten())
    return torch.cat(d)


def test_fixture_regressions_on_both_sides_of_the_switch():
    d = torch.cat([_sides(*MG.make_batch(n)[:4]) for n in MG.BATCHES])
    assert (d <= 1.0 / 9.0).sum() > 20 and (d > 1.0 / 9.0).sum() > 20


def _well_separated_batch(seed, H=128, W=160, B=2, K=6):
    """inputs with no anchor within 1e-4 of an IoU threshold, no probability near the clamp, no |t - r| near 1/9"""
    g = torch.Generator().manual_seed(seed)
    anchors = torch.from_numpy(O.anchors_for(H, W)[0])
    _, annots = O.synthetic_batch(B, size=max(H, W), G=6, num_classes=K, seed=seed)
    cls = 0.05 + 0.9 * torch.rand(B, anchors.shape[0], K, generator=g)
    reg = torch.randn(B, anchors.shape[0], 4, generator=g) * 0.3
    for b in range(B):
        _, m = assign_ref(anchors, annots[b])
        assert float(torch.minimum((m - 0.4).abs(), (m - 0.5).abs()).min()) > 1e-4
    d = _sides(cls, reg, anchors, annots)
    assert float((d - 1.0 / 9.0).abs().min()) > 1e-4
    return cls, reg, anchors, annots


@pytest.mark.parametrize('alpha,gamma', [(0.25, 2.0), (0.5, 1.5)])
def test_closed_form_gradient_equals_autograd(alpha, gamma):
    """the restatement's closed-form gradients against autograd through the oracle's FocalLoss run in fp64"""
    cls, reg, anchors, annots = _well_separated_batch(3)
    gout = (1.5, 0.5)
    ref = focal_ref(cls, reg, anchors, annots, alpha, gamma, gout)
    cr, rr = cls.double().requires_grad_(True), reg.double().requires_grad_(True)
    lc, lr = O.focal_loss(cr, rr, anchors.double()[None], annots.double(), alpha=alpha, gamma=gamma)
    torch.autograd.backward([lc, lr], [torch.tensor([gout[0]], dtype=torch.float64),
                                       torch.tensor([gout[1]], dtype=torch.float64)])
    assert min(ref['npos']) > 0
    assert rel(ref['loss'][0], lc.item()) < 1e-6 and rel(ref['loss'][1], lr.item()) < 1e-6
    # 1 - pc and t are fp32 in the restatement and fp64 here: a few fp32 ulps of the factors they enter
    assert excess(ref['dcls'], cr.grad, 1e-5 * cr.grad.abs()) <= 1.0
    # t is rounded in fp32 in the restatement and not here; the centre offsets cancel, so its error is absolute: a few
    # ulps of the coordinates (< 3e-5 here) over the anchor size (>= 22.6) and 0.1, under 1e-4
    for b in range(cls.shape[0]):
        gr = grad_scales(cls.shape[0], ref['npos'][b], gout)[1]
        assert excess(ref['dreg'][b], rr.grad[b], 1e-5 * rr.grad[b].abs() + 9 * gr * 1e-4) <= 1.0
    assert (ref['dreg'] == 0).equal(rr.grad == 0)
    assert (ref['dcls'] == 0).equal(cr.grad == 0)


def test_loss_value_misses_one_anchor_that_gradients_catch():
    """negative control of the loss-value comparison: one background anchor turned ignored at 512^2, K = 80 moves the
    loss by under the 5e-5 the loss is held to, but fails the per-element gradient bound"""
    H = W = 512
    K = 80
    g = torch.Generator().manual_seed(3)
    anchors = torch.from_numpy(O.anchors_for(H, W)[0])
    _, annots = O.synthetic_batch(1, size=H, G=8, num_classes=K, seed=0)
    cls = torch.rand(1, anchors.shape[0], K, generator=g) * 0.2
    reg = torch.randn(1, anchors.shape[0], 4, generator=g) * 0.3
    state, _ = assign_ref(anchors, annots[0])
    label, npos = labels_of(annots[0], state), int((state >= 0).sum())
    c, r, dc, dr, t32 = image_ref(cls[0], reg[0], anchors, annots[0], state, label, 0.25, 2.0)
    # the background anchor whose row contributes closest to the mean background row
    bg = torch.nonzero(state == -1).flatten()
    pc = torch.clamp(cls[0, bg], 1e-4, 1 - 1e-4).double()
    row = (0.75 * pc ** 2 * -torch.log(1 - pc)).sum(1)
    a = bg[torch.argmin((row - row.mean()).abs())]
    bad = state.clone()
    bad[a] = -2
    c2, r2, dc2, dr2, _ = image_ref(cls[0], reg[0], anchors, annots[0], bad, label, 0.25, 2.0)
    l1, l2 = losses_ref([c], [r], [npos]), losses_ref([c2], [r2], [npos])
    gc, gr = grad_scales(1, npos, (1.0, 1.0))
    print('one background anchor -> ignored: loss moves by %.2e relative' % rel(l2[0], l1[0]))
    assert rel(l2[0], l1[0]) < LOSS_RTOL
    assert excess((gc * dc2).float(), gc * dc, DCLS_RTOL * (gc * dc).abs()) > 1.0


@pytest.mark.parametrize('where', ['dcls_ignored', 'dcls_target', 'dcls_inf', 'dreg_padding_image', 'dreg_positive',
                                   'csum', 'rsum', 'loss_reg'])
def test_non_finite_output_fails_its_comparison(where):
    """negative control of every comparison against a NaN or inf in the kernels' output: the restatement itself stands in
    for the kernels and passes; one non-finite value, also where the reference is exactly 0 or in the second of the two
    losses, must fail the comparison it enters"""
    cls, reg, anchors, annots, _ = MG.make_batch('k20')
    ref = focal_ref(cls, reg, anchors, annots, gout=(1.5, 0.5))
    out = dict(state=ref['state'], npos=ref['npos'], csum=list(ref['csum']), rsum=list(ref['rsum']),
               loss=list(ref['loss']), dcls=ref['dcls'].float(), dreg=ref['dreg'].float())
    assert within(compare(out, cls, reg, anchors, annots)) == []
    state, nan = ref['state'], float('nan')
    pos = torch.nonzero(state[0] >= 0).flatten()
    if where == 'dcls_ignored':
        out['dcls'][0, torch.nonzero(state[0] == -2).flatten()[0]] = nan
    elif where == 'dcls_target':
        a = pos[0]
        out['dcls'][0, a, labels_of(annots[0], state[0])[a]] = nan
    elif where == 'dcls_inf':
        out['dcls'][1, 0, 0] = float('inf')
    elif where == 'dreg_padding_image':
        assert bool((state[2] == -3).all())
        out['dreg'][2] = nan
    elif where == 'dreg_positive':
        out['dreg'][0, pos[0], 2] = nan
    elif where == 'loss_reg':
        out['loss'][1] = nan
    else:
        out[where][1] = nan
    bad = within(compare(out, cls, reg, anchors, annots))
    assert bad == [where.split('_')[0] if not where.startswith('loss') else 'loss'], bad


def test_annotation_table_bound_is_checked_before_any_launch():
    """G = 257 is refused by argument validation, before the device is touched; G = 256 (kMaxG) passes validation and,
    without a GPU, gets as far as the CUDA error"""
    from models import _native
    _native.build()
    lib = _native.load()

    def err():
        return lib.effdet_last_error().decode()

    fake = 1 << 20                                           # aligned non-null "pointer"; never dereferenced
    for fn, extra in ((lib.effdet_focal_loss_fwd, ()), (lib.effdet_focal_loss_bwd, (fake, fake))):
        assert fn(fake, fake, fake, fake, fake, fake, fake, *extra, 2, 100, 20, 257, 0.25, 2.0, 0, None) == -1
        assert 'G=257' in err() and '256' in err()
        if not torch.cuda.is_available():
            assert fn(fake, fake, fake, fake, fake, fake, fake, *extra, 2, 100, 20, 256, 0.25, 2.0, 0, None) < 0
            assert 'G=256' not in err() and 'cuda' in err().lower()


# ------------------------------------------------------------------------------------------------
# GPU: the kernels, called the way FocalLossFn calls them, with assign_ws and stats_ws read back
# ------------------------------------------------------------------------------------------------

def run_kernels(cls, reg, anchors, annots, alpha=0.25, gamma=2.0, gout=(1.5, 0.5)):
    from models import _native as N
    B, A, K = cls.shape
    G = annots.shape[1]
    dev = cls.device
    losses = torch.empty(2, device=dev)
    assign = torch.empty((B, A), dtype=torch.int32, device=dev)
    stats = torch.empty((B, 4), device=dev)
    N.call('effdet_focal_loss_fwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors), N.f32(annots), N.f32(losses),
           assign.data_ptr(), N.f32(stats), B, A, K, G, float(alpha), float(gamma))
    g = torch.tensor(gout, dtype=torch.float32, device=dev)
    dcls, dreg = torch.empty_like(cls), torch.empty_like(reg)
    N.call('effdet_focal_loss_bwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors), N.f32(annots), N.f32(g),
           assign.data_ptr(), N.f32(stats), N.f32(dcls), N.f32(dreg), B, A, K, G, float(alpha), float(gamma))
    torch.cuda.synchronize()
    st = stats.cpu().double()
    return dict(state=assign, npos=[int(v) for v in st[:, 0]], csum=st[:, 1].tolist(), rsum=st[:, 2].tolist(),
                loss=losses.cpu().double().tolist(), dcls=dcls, dreg=dreg)


def _dev():
    return torch.device('cuda:0')


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(MG.BATCHES))
def test_kernels_match_reference_fixture(golden, name):
    cls, reg, anchors, annots, _ = MG.make_batch(name)
    p = name + '/'
    gout = tuple(golden['gout'].tolist())
    d = _dev()
    out = run_kernels(cls.to(d), reg.to(d), anchors.to(d), annots.to(d), gout=gout)
    assert np.array_equal(out['state'].cpu().numpy(), golden[p + 'state'])
    assert out['npos'] == golden[p + 'npos'].tolist()
    B = cls.shape[0]
    m = dict(loss=worst(*(rel(out['loss'][i], float(golden[p + 'losses'][i])) for i in range(2))), dcls=0.0, dreg=0.0)
    for b in range(B):
        state = torch.from_numpy(golden[p + 'state'][b])
        *_, t32 = image_ref(cls[b], reg[b], anchors, annots[b], state, labels_of(annots[b], state), 0.25, 2.0)
        rc, rr = torch.from_numpy(golden[p + 'dcls'][b]).double(), torch.from_numpy(golden[p + 'dreg'][b]).double()
        gr = grad_scales(B, out['npos'][b], gout)[1]
        m['dcls'] = worst(m['dcls'], excess(out['dcls'][b].cpu(), rc, DCLS_RTOL * rc.abs()))
        m['dreg'] = worst(m['dreg'], excess(out['dreg'][b].cpu(), rr, dreg_bound(rr, t32, gr)))
    print('%s kernels vs reference: %s' % (name, m))
    assert m['loss'] <= LOSS_RTOL and m['dcls'] <= 1.0 and m['dreg'] <= 1.0, m


def _geometry(case):
    """(cls, reg, anchors, annots) on the device for one geometry; synthetic annotations as bench.py makes them, or
    K-class crafted boundary images"""
    name, H, W, B, K = case
    d = _dev()
    anchors = torch.from_numpy(O.anchors_for(H, W)[0])
    rng = np.random.RandomState(B * 1000 + K)
    G = MG.G_ROWS
    if name == 'full_table':
        annots = np.stack([MG.table(MG.random_rows(rng, 256, H, W, K), 256) for _ in range(B)])
    else:
        _, syn = O.synthetic_batch(B, size=H, G=8, num_classes=K, seed=0)       # bench.py's synthetic annotations
        annots = np.full((B, G, 5), -1.0, np.float32)
        annots[:, :8] = syn.numpy()
        for b, plan in zip((B - 2, B - 1), MG.plans(K)):                        # the last two: crafted images
            annots[b] = MG.crafted_image(anchors.numpy(), H, W, K, plan, rng, G)[0]
    g = torch.Generator(device=d).manual_seed(B * 7 + K)
    A = anchors.shape[0]
    cls = torch.rand(B, A, K, generator=g, device=d) * 0.2
    flat = cls.view(-1)
    idx = torch.arange(0, flat.numel(), 1009, device=d)     # sparse: near-1 values dominate a sum at p ~ U(0, 0.2)
    flat[idx] = torch.from_numpy(MG.SPECIAL_P).to(d)[idx % MG.SPECIAL_P.size]
    reg = torch.randn(B, A, 4, generator=g, device=d) * 0.3
    return cls, reg, anchors.to(d), torch.from_numpy(annots).to(d)


GEOMETRIES = [('d0', 512, 512, 32, 80), ('d4', 1024, 1024, 4, 80), ('k1', 512, 512, 2, 1), ('k3', 512, 512, 2, 3),
              ('k20', 512, 512, 2, 20), ('k90', 512, 512, 2, 90), ('full_table', 512, 512, 2, 20),
              ('non_square', 384, 640, 2, 20)]


RUNS = [(c, (1.5, 0.5)) for c in GEOMETRIES] + [(c, (0.0, 1.0)) for c in GEOMETRIES if c[0] in ('k3', 'k20')]


@pytest.mark.gpu
@pytest.mark.parametrize('case,gout', RUNS, ids=['%s-gout%g,%g' % (c[0], *g) for c, g in RUNS])
def test_kernels_match_restatement(case, gout):
    cls, reg, anchors, annots = _geometry(case)
    out = run_kernels(cls, reg, anchors, annots, gout=gout)
    m = compare(out, cls, reg, anchors, annots, gout=gout)
    print('%s %s: %s, positives %s' % (case[0], gout, m, out['npos'][:8]))
    assert not within(m), m
    if gout[0] == 0:
        assert bool((out['dcls'] == 0).all())


@pytest.mark.gpu
def test_every_comparison_catches_its_fault():
    """negative controls: the reference of image 0 with one flipped state, one swapped label or a positive count off by
    one exceeds each comparison's bound at least once; the uncorrupted reference passes"""
    case = ('k20', 512, 512, 2, 20)
    cls, reg, anchors, annots = _geometry(case)
    out = run_kernels(cls, reg, anchors, annots)
    assert not within(compare(out, cls, reg, anchors, annots))
    caught = {}
    for fault in ('state', 'label', 'npos'):
        m = compare(out, cls, reg, anchors, annots, fault=fault)
        print('fault %s: %s' % (fault, m))
        caught[fault] = set(within(m))
    assert {'state', 'csum', 'rsum', 'dcls', 'dreg'} <= caught['state']
    assert 'dcls' in caught['label']
    assert {'npos', 'loss', 'dcls', 'dreg'} <= caught['npos']
    assert set().union(*caught.values()) == {'state', 'npos', 'csum', 'rsum', 'loss', 'dcls', 'dreg'}


@pytest.mark.gpu
@pytest.mark.parametrize('used', ['cls', 'reg'])
def test_focal_loss_module_with_one_loss_used(used):
    """through models.losses.FocalLoss under autograd, only one of the two losses used: autograd hands backward a zero
    upstream gradient for the unused output (gradients are materialised), and that output's gradient tensor must be
    exactly zero.  FocalLossFn.backward also takes None for an absent upstream gradient; called directly with None it
    must give the same gradients bit for bit."""
    from models.losses import FocalLoss
    cls, reg, anchors, annots = _geometry(('k20', 512, 512, 2, 20))
    cd, rd = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    lc, lr = FocalLoss()(cd, rd, anchors[None], annots)
    ((lc if used == 'cls' else lr) * 1.5).backward()
    gout = (1.5, 0.0) if used == 'cls' else (0.0, 1.5)
    m = compare(dict(loss=[lc.item(), lr.item()], dcls=cd.grad, dreg=rd.grad), cls, reg, anchors, annots, gout=gout)
    print('FocalLoss, %s loss only: %s' % (used, m))
    assert not within(m), m
    assert bool(((rd.grad if used == 'cls' else cd.grad) == 0).all())
    from models._ops import FocalLossFn

    class Ctx:
        def save_for_backward(self, *tensors):
            self.saved_tensors = tensors

    ctx = Ctx()
    FocalLossFn.forward(ctx, cls, reg, anchors[None], annots, 0.25, 2.0)
    g = torch.tensor([1.5], device=cls.device)
    dcls, dreg = FocalLossFn.backward(ctx, *((g, None) if used == 'cls' else (None, g)))[:2]
    assert torch.equal(dcls, cd.grad) and torch.equal(dreg, rd.grad)


@pytest.mark.gpu
def test_focal_loss_module_general_alpha_gamma():
    """FocalLoss with gamma = 1.5, alpha = 0.5: the powf path of the kernels"""
    from models.losses import FocalLoss
    cls, reg, anchors, annots = _geometry(('k20', 512, 512, 2, 20))
    fl = FocalLoss()
    fl.alpha, fl.gamma = 0.5, 1.5
    cd, rd = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    lc, lr = fl(cd, rd, anchors[None], annots)
    torch.autograd.backward([lc, lr], [torch.tensor([1.5], device=cls.device), torch.tensor([0.5], device=cls.device)])
    m = compare(dict(loss=[lc.item(), lr.item()], dcls=cd.grad, dreg=rd.grad), cls, reg, anchors, annots,
                alpha=0.5, gamma=1.5, gout=(1.5, 0.5))
    print('FocalLoss alpha 0.5 gamma 1.5: %s' % m)
    assert not within(m), m
