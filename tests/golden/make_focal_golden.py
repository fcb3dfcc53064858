"""Pin the FocalLoss kernels' anchor assignment, losses and gradients against the reference's OWN loss code.  calc_iou
and FocalLoss are cut out of the reference's models/losses.py with `ast` and executed unmodified on the CPU, with
torch.Tensor.cuda bound to the identity for the duration of the run; the gradients are taken by autograd through that
code with an upstream gradient of (1.5, 0.5).  Output -> tests/golden/focal_loss.npz.

Two batches at 128 x 192 (A = 4,608 anchors): K = 20 (the kernels' 4-wide path) and K = 3 (the scalar path).  The
inputs are regenerated from seeds by make_batch(), which the tests import, so the file holds per batch the annotations,
the reference's per-anchor state in the kernel's encoding (the unfiltered annotation row of a positive anchor, -1
background, -2 ignored, -3 no annotations), IoU_max at the crafted anchors, the positive counts, the two losses and the
gradients in fp32.

The crafted cases, each at least once over the two batches: anchors at an IoU of exactly 0.5f and 0.4f, and one and two
fp32 ulps either side of both; two annotation rows tied at an anchor's maximum IoU with different labels (a duplicated
box, and two distinct boxes mirrored about the anchor), the first of which must win; padding rows between real rows; an
image whose annotations give no positive anchor and an image with only padding rows; a zero-width box, a sub-pixel box
and a box partly outside the image; class probabilities at float32(1e-4) and float32(0.9999), one ulp either side of
each and outside the clamp, on target and non-target entries; regressions on both sides of |target - regression| = 1/9.

Crafted anchors are the level-3, ratio-1, scale-1 anchors [8gx-12, 8gy-12, 8gx+20, 8gy+20] (32 x 32, integer corners):
half of one has an IoU of exactly 0.5 with it, and a 40 x 64 box containing it one of exactly 0.4.  The near-threshold
boxes step two corners of those boxes one fp32 ulp at a time until the IoU, in the reference's fp32 arithmetic, is the
wanted neighbour of the threshold.  Slots sit 56 px apart in x and 72 px in y, so no box reaches another slot's anchor.

usage: python tests/golden/make_focal_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
import itertools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'oracle'))
import effdet_oracle as O  # noqa: E402

SIZE = (128, 192)
BATCHES = {'k20': (20, 3, 31), 'k3': (3, 4, 32)}           # name: (K, B, seed)
G_ROWS = 24
GOUT = (1.5, 0.5)
P_LO, P_HI = np.float32(1e-4), np.float32(1.0 - 1e-4)     # the clamp bounds as the reference's fp32 tensor sees them


def ulps(v, n):
    """v stepped n fp32 ulps (n < 0: downwards)"""
    v = np.float32(v)
    for _ in range(abs(n)):
        v = np.nextafter(v, np.float32(np.inf if n > 0 else -np.inf))
    return v


# class probabilities at and around the clamp bounds, and outside them
SPECIAL_P = np.array([P_LO, ulps(P_LO, -1), ulps(P_LO, 1), P_HI, ulps(P_HI, -1), ulps(P_HI, 1), 0.0, 2e-5, 0.99995, 1.0],
                     np.float32)
# regression - target offsets: |.| below, at about, and above the smooth-L1 switch 1/9
REG_OFFSETS = np.array([0.05, -0.1, 0.11, -0.112, 0.3, -2.0], np.float32)


def slot_anchor(anchors, W, gx, gy):
    """index of the level-3 ratio-1 scale-1 anchor of grid cell (gx, gy) and its box"""
    a = (gy * ((W + 7) // 8) + gx) * 9 + 3
    box = [8.0 * gx - 12, 8.0 * gy - 12, 8.0 * gx + 20, 8.0 * gy + 20]
    assert anchors[a].tolist() == box, (a, anchors[a], box)
    return a, box


def near_box(anchor, box, thr, n):
    """box stepped at two corners until its fp32 IoU with anchor is thr stepped n ulps; the first hit in a fixed
    order, so the result is reproducible"""
    want = ulps(thr, n)
    if n == 0:
        assert O.pairwise_iou(torch.tensor([anchor]), torch.tensor([box]))[0, 0].item() == want
        return list(box)
    span = np.arange(-48, 49)
    for i, j in itertools.combinations(range(4), 2):
        ci = np.array([ulps(box[i], s) for s in span], np.float32)
        cj = np.array([ulps(box[j], s) for s in span], np.float32)
        bx = np.tile(np.array(box, np.float32), (span.size * span.size, 1))
        bx[:, i], bx[:, j] = np.repeat(ci, span.size), np.tile(cj, span.size)
        v = O.pairwise_iou(torch.tensor([anchor], dtype=torch.float32), torch.from_numpy(bx))[0].numpy()
        hit = np.nonzero(v == want)[0]
        if hit.size:
            return bx[hit[0]].tolist()
    raise AssertionError('no box at IoU %r' % want)


def slot_rows(anchors, W, gx, gy, kind, labels):
    """annotation rows ([x1, y1, x2, y2, label] or None for a padding row) of one slot, and the crafted anchor as
    (anchor index, kind, wanted IoU or None)"""
    a, an = slot_anchor(anchors, W, gx, gy)
    x0, y0 = an[0], an[1]
    if kind[0] == 'iou':
        thr, n = kind[1], kind[2]
        base = [x0, y0, x0 + 16, y0 + 32] if thr == 0.5 else [x0 - 8, y0 - 8, x0 + 32, y0 + 56]
        return [near_box(an, base, thr, n) + [labels[0]]], (a, 'iou%.1f%+d' % (thr, n), ulps(thr, n))
    if kind[0] == 'tie_duplicate':                          # the same box twice, a padding row between
        return [an + [labels[0]], None, an + [labels[1]]], (a, 'tie_duplicate', np.float32(1.0))
    if kind[0] == 'tie_mirror':                             # two boxes mirrored about the anchor's vertical axis
        return ([[x0 - 4, y0, x0 + 28, y0 + 32, labels[0]], [x0 + 4, y0, x0 + 36, y0 + 32, labels[1]]],
                (a, 'tie_mirror', np.float32(896.0 / 1152.0)))
    raise ValueError(kind)


def spaced(rows):
    """rows with a padding row (None) after every second one"""
    out = []
    for i, r in enumerate(rows):
        out += [r, None] if i % 2 == 1 else [r]
    return out


def table(rows, G):
    t = np.full((G, 5), -1.0, np.float32)
    assert len(rows) <= G
    for i, r in enumerate(rows):
        if r is not None:
            t[i] = r
    return t


def random_rows(rng, n, H, W, K):
    rows = []
    for _ in range(n):
        x, y = rng.uniform(-8, W - 24), rng.uniform(-8, H - 24)
        w, h = rng.uniform(16, 96, size=2)
        rows.append([x, y, x + w, y + h, float(rng.randint(K))])
    return rows


def crafted_image(anchors, H, W, K, plan, rng, G):
    """an annotation table for the slots in plan ({(gx, gy): kind}), with a padding row after every second real row,
    and the crafted anchors"""
    rows, crafted = [], []
    for (gx, gy), kind in plan.items():
        labels = rng.choice(K, size=2, replace=False).astype(np.float64).tolist() if K > 1 else [0.0, 0.0]
        if kind[0] == 'rows':
            rows += kind[1]
            continue
        r, c = slot_rows(anchors, W, gx, gy, kind, labels)
        rows += r
        crafted.append(c)
    return table(spaced(rows), G), crafted


SLOTS = [(0, 0), (7, 0), (14, 0), (21, 0), (0, 9), (7, 9), (14, 9), (21, 9)]


def plans(K):
    """the crafted images of a batch at 128 x 192; 'rows' entries are plain annotation rows"""
    thresholds_a = dict(zip(SLOTS, [('iou', 0.5, 0), ('iou', 0.4, 0), ('iou', 0.5, -2), ('iou', 0.5, -1),
                                    ('iou', 0.5, 1), ('iou', 0.5, 2), ('tie_duplicate',), ('tie_mirror',)]))
    thresholds_b = dict(zip(SLOTS[:4], [('iou', 0.4, -2), ('iou', 0.4, -1), ('iou', 0.4, 1), ('iou', 0.4, 2)]))
    thresholds_b[(0, 9)] = ('rows', [[-4.0, 64.0, -4.0, 84.0, 0.0],            # zero width
                                     [40.0, 70.0, 40.4, 70.3, float(K - 1)],   # sub-pixel: clamp(min=1) of both sides
                                     [150.0, 80.0, 215.0, 140.0, 0.0],        # partly outside the image
                                     [100.0, 70.0, 140.0, 110.0, float(K // 2)]])
    return thresholds_a, thresholds_b


def make_batch(name):
    """-> (cls [B,A,K] f32, reg [B,A,4] f32, anchors [A,4] f32, annots [B,G,5] f32, crafted) regenerated from the
    batch's seed; crafted is a list of (image, anchor, kind, wanted IoU)"""
    K, B, seed = BATCHES[name]
    H, W = SIZE
    rng = np.random.RandomState(seed)
    anchors = O.anchors_for(H, W)[0]
    pa, pb = plans(K)
    tiny = [[x, y, x + 2.0, y + 2.0, float(k % K)] for k, (x, y) in enumerate([(10, 10), (90, 40), (170, 100)])]
    if name == 'k20':
        images = [('crafted', pa), ('crafted', pb), ('padding', None)]
    else:
        images = [('rows', tiny), ('crafted', pa), ('crafted', pb), ('rows', random_rows(rng, 6, H, W, K))]
    annots, crafted = [], []
    for b, (what, arg) in enumerate(images):
        if what == 'crafted':
            t, c = crafted_image(anchors, H, W, K, arg, rng, G_ROWS)
            crafted += [(b, a, kind, v) for a, kind, v in c]
        elif what == 'rows':
            t = table(spaced(arg), G_ROWS)
        else:
            t = table([], G_ROWS)
        annots.append(t)
    annots = np.stack(annots)
    A = anchors.shape[0]
    cls = rng.uniform(0.0, 0.3, size=(B, A, K)).astype(np.float32)
    reg = (rng.standard_normal((B, A, 4)) * 0.3).astype(np.float32)
    # special probabilities on target entries of positive anchors, on every anchor's entries in a stripe, and
    # regression offsets around 1/9 on positive anchors
    an = torch.from_numpy(anchors)
    for b in range(B):
        valid = np.nonzero(annots[b, :, 4] != -1)[0]
        if valid.size == 0:
            continue
        gt = torch.from_numpy(annots[b, valid])
        m, arg = torch.max(O.pairwise_iou(an, gt[:, :4]), dim=1)
        pos = torch.nonzero(m >= 0.5).flatten().numpy()
        for i, a in enumerate(pos):
            lab = int(gt[arg[a], 4])
            cls[b, a, lab] = SPECIAL_P[(i + b) % SPECIAL_P.size]
            g = gt[arg[a]]
            aw, ah = an[a, 2] - an[a, 0], an[a, 3] - an[a, 1]
            gw, gh = g[2] - g[0], g[3] - g[1]
            t = torch.stack([((g[0] + 0.5 * gw) - (an[a, 0] + 0.5 * aw)) / aw,
                             ((g[1] + 0.5 * gh) - (an[a, 1] + 0.5 * ah)) / ah,
                             torch.log(torch.clamp(gw, min=1) / aw), torch.log(torch.clamp(gh, min=1) / ah)])
            t = (t / torch.tensor([0.1, 0.1, 0.2, 0.2])).numpy()
            reg[b, a] = t + REG_OFFSETS[(np.arange(4) + i) % REG_OFFSETS.size]
        stripe = np.arange(b, A, 7)
        cls[b, stripe] = SPECIAL_P[(stripe[:, None] + np.arange(K)[None]) % SPECIAL_P.size]
    return (torch.from_numpy(cls), torch.from_numpy(reg), torch.from_numpy(anchors), torch.from_numpy(annots), crafted)


if __name__ == '__main__':
    import ast
    REF = os.environ.get('EFFDET_REFERENCE')          # path of a checkout of the reference repository
    assert REF, 'set EFFDET_REFERENCE to a checkout of the reference repository'
    ns = {'np': np, 'torch': torch, 'nn': torch.nn}
    for node in ast.parse(open(os.path.join(REF, 'models', 'losses.py')).read()).body:
        if getattr(node, 'name', None) in {'calc_iou', 'FocalLoss'}:
            exec(compile(ast.Module([node], []), 'losses.py', 'exec'), ns)
    out = {'size': np.array(SIZE), 'gout': np.array(GOUT, np.float32)}
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for name in BATCHES:
            cls, reg, anchors, annots, crafted = make_batch(name)
            B, A, K = cls.shape
            cr, rr = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
            lc, lr = ns['FocalLoss']()(cr, rr, anchors[None], annots)
            torch.autograd.backward([lc, lr], [torch.tensor([GOUT[0]]), torch.tensor([GOUT[1]])])
            # the assignment as FocalLoss.forward makes it (losses.py:52, 63-76), from the reference's calc_iou
            state = np.full((B, A), -3, np.int32)
            iou_max = np.zeros((B, A), np.float32)
            for b in range(B):
                rows = torch.nonzero(annots[b, :, 4] != -1).flatten()
                if rows.numel() == 0:
                    continue
                m, arg = torch.max(ns['calc_iou'](anchors, annots[b, rows, :4]), dim=1)
                s = torch.where(torch.ge(m, 0.5), rows[arg], torch.full_like(rows[arg], -2))
                s[torch.lt(m, 0.4)] = -1
                state[b], iou_max[b] = s.numpy(), m.numpy()
            npos = (state >= 0).sum(1).astype(np.int32)
            ocl, orl = O.focal_loss(cls, reg, anchors[None], annots)
            assert torch.equal(ocl, lc.detach()) and torch.equal(orl, lr.detach()), 'oracle != reference losses'
            cb, ca = np.array([c[0] for c in crafted]), np.array([c[1] for c in crafted])
            assert np.array_equal(iou_max[cb, ca], np.array([c[3] for c in crafted], np.float32)), 'crafted IoU'
            p = name + '/'
            out.update({p + 'annots': annots.numpy(), p + 'state': state, p + 'npos': npos,
                        p + 'crafted_image': cb.astype(np.int32), p + 'crafted_anchor': ca.astype(np.int32),
                        p + 'crafted_kind': np.array([c[2] for c in crafted]), p + 'crafted_iou': iou_max[cb, ca],
                        p + 'losses': np.array([lc.item(), lr.item()], np.float32),
                        p + 'dcls': cr.grad.numpy(), p + 'dreg': rr.grad.numpy()})
            print('%s: K=%d B=%d A=%d, positives %s, losses %.8g %.8g, crafted %s'
                  % (name, K, B, A, npos.tolist(), lc.item(), lr.item(), [c[2] for c in crafted]))
    finally:
        torch.Tensor.cuda = cuda
    np.savez_compressed(os.path.join(HERE, 'focal_loss.npz'), **out)
    print('focal_loss.npz written: %d bytes' % os.path.getsize(os.path.join(HERE, 'focal_loss.npz')))
