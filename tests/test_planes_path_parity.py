"""Kernel-level fp64 parity of the bf16x3 planes path: the RetinaHead and BiFPN 3x3 layers of the train step.

  wgrad_tc2_multi_kernel  weight gradient of all pyramid levels in one launch (wgrad_planes_multi)
  to_planes_kernel        fp32 -> bf16 hi/lo planes, with the sigmoid backward and the bias gradient folded in
  conv_planes_kernel      the head's output convs (strided slices of the concatenated outputs) and data gradients
  fuse_fwd_kernel, fuse_bwd_{up,pool}_kernel, fuse_bwd_weights_kernel   BiFPN fast-normalised fusion

The module tests hold parameter gradients to 5e-3 .. 5e-2 because ReLU masks flip between the CPU and GPU summation
orders.  Here every kernel gets its own inputs, so nothing can flip and the bounds are tight.  Every reference is
float64 on the CPU, built from the same fp32 operands with F.conv2d, F.conv_transpose2d, torch.nn.grad.conv2d_weight and
F.max_pool2d.

Bounds:
  TOL_TC    = 3e-5  whole-tensor norm-relative error of a bf16x3 tensor-core output (three bf16 products per
                    multiply-add, fp32 accumulation; ~1e-5 is typical), weight gradients included: their launcher
                    caps the pixel chunks one CTA accumulates (kWgMaxChunksPerSplit, conv_tc.cu), without which
                    the error grew linearly with that K range (3.8e-5 at 171 chunks)
  TOL_LOCAL = 1e-4  the same metric on every block of 64 output channels x tap of a weight gradient, and on every pyramid
                    level of a forward or data-gradient output.  A whole-tensor norm averages an error confined to one
                    tile away; the smaller blocks scatter more around the bf16x3 noise, so they get 3x headroom, and stay
                    3x below what one bf16 product per multiply-add gives (> 3e-4: operands rounded to 8 bits).  A tile
                    computed with one product, a dropped level (> 5e-2 of a block here) or a missing chunk fails it.
  TOL_EXACT = 5e-6  fp32 kernels without a reduction (fusion values and data gradients)
  TOL_SUM   = 2e-5  fp32 sums over up to 10^7 elements that thousands of blocks add with atomics (column sums, the
                    fusion-weight gradient): ~2^-24 * sqrt(blocks) relative, a few 1e-6 at the sizes here
Each test also runs a negative control that shows its bound has teeth."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

TOL_TC = 3e-5
TOL_LOCAL = 1e-4
TOL_EXACT = 5e-6
TOL_SUM = 2e-5
SINGLE_PASS_MIN = 3e-4          # what one bf16 product per multiply-add must exceed

A = 9                           # anchors per pixel
# pyramid levels P3..P7 (H, W) of the head, for the image sizes whose every level has a TMA pixel box
LEVEL_SETS = {
    'd0_512': [(64, 64), (32, 32), (16, 16), (8, 8), (4, 4)],
    'd4_1024': [(128, 128), (64, 64), (32, 32), (16, 16), (8, 8)],
    'wide_1024x512': [(128, 64), (64, 32), (32, 16), (16, 8), (8, 4)],
}
# D7 (1536^2): its 96x96 level has no pixel box, so the head of D7 runs the gathering kernels, never the planes path
D7_1536 = [(192, 192), (96, 96), (48, 48), (24, 24), (12, 12)]
# (Cin, Cout) of the model's 3x3 layers: D0 tower / box / class (20 classes), D1 BiFPN, D4 class (80 classes),
# D5 class (80 classes), D7 tower.  With 90 classes the class conv has 810 outputs, not a multiple of 4: it is refused
# by the tensor-core packs and never runs here (test_level_sets_have_pixel_boxes).
WGRAD_PAIRS = [(64, 64), (64, 36), (64, 180), (88, 88), (224, 720), (288, 720), (384, 384)]


def _dev():
    return torch.device('cuda:0')


def _cdiv(a, b):
    return -(-a // b)


@pytest.fixture()
def ops():
    from models import _ops
    old = _ops.PRECISION
    _ops.PRECISION = 'bf16x3'
    yield _ops
    _ops.PRECISION = old


class _single_pass:
    """one bf16 product per multiply-add (tc_single = 1) for the launches inside the block"""

    def __init__(self, ops):
        self.ops = ops

    def __enter__(self):
        self.old, self.ops.PRECISION = self.ops.PRECISION, 'bf16'

    def __exit__(self, *exc):
        self.ops.PRECISION = self.old


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, generator=g)


def _rel(got, want):
    return O.rel_err(got, want)


# ------------------------------------------------------------------------------------------------
# pixel boxes and split-K: mirrors of wg_geometry and wgrad_tc2_launch (conv_tc.cu)
# ------------------------------------------------------------------------------------------------

WG_MAX_CHUNKS_PER_SPLIT = 64    # kWgMaxChunksPerSplit


def _box(B, H, W):
    """(images per pixel box Bb, image boxes nbb) of one level, or None when it has no box"""
    Wb = W if W <= 64 else 64
    if W % Wb:
        return None
    Hb = max(h for h in range(1, H + 1) if H % h == 0 and Wb * h <= 64)
    Bb = min(max(64 // (Wb * Hb), 1), B)
    ks = Wb * Hb * Bb
    if ks < 16 or ks % 16:
        return None
    return Bb, _cdiv(B, Bb)


def _chunks(B, H, W):
    """pixel boxes (GEMM-K chunks) of one level, or None when it has no box"""
    box = _box(B, H, W)
    if box is None:
        return None
    Wb = W if W <= 64 else 64
    Hb = max(h for h in range(1, H + 1) if H % h == 0 and Wb * h <= 64)
    return (W // Wb) * (H // Hb) * box[1]


def _split_plan(B, levels, Cin, Cout, sms, cap=WG_MAX_CHUNKS_PER_SPLIT):
    """(first chunk of every level, chunks, chunks_per_split, splits) of one wgrad_tc2_multi_kernel launch, as
    wgrad_tc2_launch computes them (cap=None: without the cap on chunks per split)"""
    begins, n = [], 0
    for h, w in levels:
        begins.append(n)
        n += _chunks(B, h, w)
    ct, nt = _cdiv(Cin, 256 if Cin > 64 else 64), _cdiv(Cout, 128)
    splits = max(1, (sms * 2) // (ct * nt * 9))
    splits = min(splits, _cdiv(n, 4))
    if cap is not None:
        splits = max(splits, _cdiv(n, cap))
    cps = _cdiv(n, splits)
    return begins, n, cps, _cdiv(n, cps)


def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


def _split_cases(B, levels, Cin, Cout, sms):
    """which split-K placements the launches of test_wgrad_planes_multi produce (each level alone, then all levels)"""
    found = set()
    for ls in [[lv] for lv in levels] + [levels]:
        begins, n, cps, splits = _split_plan(B, ls, Cin, Cout, sms)
        if splits == 1 and cps > 1:
            found.add('one split')
        if cps == 1:
            found.add('one chunk per split')
        if len(ls) > 1:
            ends = begins[1:] + [n]
            inside = any(b0 < k * cps < e for k in range(1, splits) for b0, e in zip(begins, ends))
            straddle = any(s * cps < b0 < (s + 1) * cps for s in range(splits) for b0 in begins[1:])
            if inside and straddle:
                found.add('boundary inside a level')
    return found


SPLIT_CASES = {'one split', 'one chunk per split', 'boundary inside a level'}


def _wgrad_batch(levels, Cin, Cout):
    sms = _sms()
    for B in range(1, 65):
        if _split_cases(B, levels, Cin, Cout, sms) == SPLIT_CASES:
            return B
    raise AssertionError('no batch produces every split-K case for %s %d->%d on %d SMs' % (levels, Cin, Cout, sms))


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_level_sets_have_pixel_boxes():
    """every level set used below has a pixel box (and the Python mirror of wg_geometry agrees with the library);
    D7 1536^2 and 90 classes stay off the planes path"""
    import __graft_entry__ as entry
    entry.build()
    from models import _native as N, _ops
    lib = N.load()
    for name, levels in LEVEL_SETS.items():
        for B in range(1, 9):
            for h, w in levels:
                assert lib.effdet_wgrad_tc_geometry_ok(B, h, w) == 1, (name, B, h, w)
                assert _chunks(B, h, w) is not None, (name, B, h, w)
    for B in (1, 2, 4):
        for h, w in D7_1536 + [(2, 2), (8, 2), (96, 32), (80, 80)]:
            assert bool(lib.effdet_wgrad_tc_geometry_ok(B, h, w)) == (_chunks(B, h, w) is not None), (B, h, w)
    assert not lib.effdet_wgrad_tc_geometry_ok(1, 96, 96)
    # the split-K mirror: chunks per level add up as the launcher counts them, and a D0 launch splits
    begins, n, cps, splits = _split_plan(1, LEVEL_SETS['d0_512'], 64, 64, 132)
    assert begins == [0, 64, 80, 84, 85] and n == 86 and (cps, splits) == (4, 22)
    assert _split_cases(1, LEVEL_SETS['d0_512'], 64, 64, 132) == SPLIT_CASES
    # the benchmarked step's class conv: 2728 chunks, 4 splits of 682 chunks without the cap, 43 of 64 with it
    assert _split_plan(32, LEVEL_SETS['d0_512'], 256, 720, 132, cap=None)[1:] == (2728, 682, 4)
    assert _split_plan(32, LEVEL_SETS['d0_512'], 256, 720, 132)[1:] == (2728, 64, 43)
    old = _ops.PRECISION
    try:
        _ops.PRECISION = 'bf16x3'
        assert _ops.tc_packs(torch.empty(810, 64, 3, 3)) == (None, None)
    finally:
        _ops.PRECISION = old


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _to_planes(ops, x):
    """fp32 [B, H, W, C] on the device -> planes [2, B, H, W, pitch]"""
    b, h, w, c = x.shape
    p = ops._planes(b, h, w, c, x)
    ops.to_planes(x.data_ptr(), h * w * c, p, b, h * w, c, x)
    return p


def _from_planes(p, C):
    return (p[0].double() + p[1].double())[..., :C].cpu()


def _nan_planes(ops, B, H, W, C):
    return torch.full((2, B, H, W, ops._pitch8(C)), float('nan'), device=_dev(), dtype=torch.bfloat16)


def _check(got, want, what, tol=TOL_TC):
    e = _rel(torch.cat([t.flatten() for t in got]), torch.cat([t.flatten() for t in want]))
    loc = max(_rel(g, w) for g, w in zip(got, want))
    print('%s: rel err %.2e (bound %.0e), worst level %.2e (bound %.0e)' % (what, e, tol, loc, TOL_LOCAL))
    assert e < tol, (what, e)
    assert loc < TOL_LOCAL, (what, loc)
    return e


# ------------------------------------------------------------------------------------------------
# 1. wgrad_tc2_multi_kernel in bf16x3
# ------------------------------------------------------------------------------------------------

def _block_errs(got, want):
    """norm-relative error of every block of 64 output channels x tap of an OIHW weight gradient"""
    Cout = want.shape[0]
    errs = []
    for n0 in range(0, Cout, 64):
        for t in range(9):
            errs.append(_rel(got[n0:n0 + 64, :, t // 3, t % 3], want[n0:n0 + 64, :, t // 3, t % 3]))
    return errs


def _check_dw(got, want, what):
    e, loc = _rel(got, want), max(_block_errs(got, want))
    print('%s: rel err %.2e (bound %.0e), worst 64-channel x tap block %.2e (bound %.0e)' % (what, e, TOL_TC, loc, TOL_LOCAL))
    assert e < TOL_TC, (what, e)
    assert loc < TOL_LOCAL, (what, loc)


def _wgrad_case(ops, levels, B, Cin, Cout, seed, what):
    """every level alone against its own fp64 reference, then all levels in one launch against the fp64 sum, each added
    to a non-zero dw; negative controls: a reference without the smallest level, one bf16 product per multiply-add"""
    assert ops.pixel_boxes_ok([(B, h, w) for h, w in levels])
    g = _gen(seed)
    xs = [_randn(g, B, h, w, Cin) for h, w in levels]
    dys = [_randn(g, B, h, w, Cout) for h, w in levels]
    xp = [_to_planes(ops, x.to(_dev())) for x in xs]
    dyp = [_to_planes(ops, d.to(_dev())) for d in dys]
    shape = (Cout, Cin, 3, 3)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    refs = [torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2).double(), shape, d.permute(0, 3, 1, 2).double(), 1, 1)
            for x, d in zip(xs, dys)]
    del xs, dys
    total = sum(refs)
    dw0 = (_randn(g, *shape) * float(total.std())).to(_dev())
    wd = torch.empty(shape, device=_dev())        # only the device of the launch

    def launch(ls, precise=True):
        dw = dw0.clone()
        lv = [dict(x=xp[i], dy=dyp[i], B=B, H=levels[i][0], W=levels[i][1]) for i in ls]
        if precise:
            ops.wgrad_planes_multi(wd, lv, dw, Cin, Cout, 3)
        else:
            with _single_pass(ops):
                ops.wgrad_planes_multi(wd, lv, dw, Cin, Cout, 3)
        return dw.double().cpu() - dw0.double().cpu()

    sms = _sms()
    for i, (h, w) in enumerate(levels):
        cps = _split_plan(B, [(h, w)], Cin, Cout, sms)[2]
        _check_dw(launch([i]), refs[i], '%s level %dx%d alone, %d chunks per split' % (what, h, w, cps))
    got = launch(range(len(levels)))
    _check_dw(got, total, '%s all levels, %d chunks per split' % (what, _split_plan(B, levels, Cin, Cout, sms)[2]))
    miss = max(_block_errs(got, total - refs[-1]))
    single = _rel(launch(range(len(levels)), precise=False), total)
    print('  controls: without the smallest level worst block %.2e, single pass %.2e' % (miss, single))
    assert miss > TOL_LOCAL and single > SINGLE_PASS_MIN, (miss, single)


@pytest.mark.gpu
@pytest.mark.parametrize('Cin,Cout', WGRAD_PAIRS)
@pytest.mark.parametrize('geo', list(LEVEL_SETS))
def test_wgrad_planes_multi(ops, geo, Cin, Cout):
    """split-K placement: B is the smallest batch whose launches (each level alone, then all levels) include, at this
    device's SM count, one split, a split boundary inside a level (a split that straddles two levels) and one chunk per
    split -- B = 1 on 114 and on 132 SMs"""
    levels = LEVEL_SETS[geo]
    B = _wgrad_batch(levels, Cin, Cout)
    _wgrad_case(ops, levels, B, Cin, Cout, Cin * 1000 + Cout + len(geo), 'wgrad %d->%d %s B=%d' % (Cin, Cout, geo, B))


@pytest.mark.gpu
@pytest.mark.parametrize('geo,B,Cin,Cout', [('d0_512', 5, 64, 64), ('d0_512', 5, 88, 88), ('wide_1024x512', 5, 64, 180),
                                            ('d0_512', 32, 256, 720), ('d0_512', 32, 256, 256)])
def test_wgrad_planes_multi_batched(ops, geo, B, Cin, Cout):
    """several images per pixel box (the image axis of the TMA box, a partial last box when B % Bb != 0), and the
    benchmarked step's head layers (D0 512^2, B = 32): their K ranges are long enough that without the cap of
    kWgMaxChunksPerSplit (conv_tc.cu) one CTA would accumulate up to 682 chunks"""
    levels = LEVEL_SETS[geo]
    boxes = [_box(B, h, w) for h, w in levels]
    assert any(nbb > 1 for _, nbb in boxes) and (B == 32 or any(B % bb for bb, _ in boxes)), boxes
    sms = _sms()
    plan, uncapped = _split_plan(B, levels, Cin, Cout, sms), _split_plan(B, levels, Cin, Cout, sms, cap=None)
    assert plan[2] <= WG_MAX_CHUNKS_PER_SPLIT and (B < 32 or uncapped[2] > 3 * WG_MAX_CHUNKS_PER_SPLIT), (plan, uncapped)
    _wgrad_case(ops, levels, B, Cin, Cout, 31 * B + Cin + Cout, 'wgrad %d->%d %s B=%d' % (Cin, Cout, geo, B))


# ------------------------------------------------------------------------------------------------
# 2. to_planes_kernel
# ------------------------------------------------------------------------------------------------

def _head_layout(levels, width, gap=2):
    """offsets (in pixels x anchors) of the levels in a concatenated [B, tot, width] head output, with `gap` unused
    pixels before, between and after the levels (they must never be read or written)"""
    offs, tot = [], gap * A
    for h, w in levels:
        offs.append(tot)
        tot += h * w * A + gap * A
    return offs, tot


def _slice(t, off, h, w, width):
    B = t.shape[0]
    return t[:, off:off + h * w * A, :].reshape(B, h, w, A * width)


def _bits(t):
    return t.contiguous().view(torch.int16)


# (C, width per anchor or None for a dense [B, H, W, C] source, with the sigmoid backward, level set, B)
TO_PLANES_CASES = [
    (36, 4, False, 'd0_512', 256),       # box conv gradient; the 64x64 level has 1M rows: many blocks add atomically
    (180, 20, True, 'wide_1024x512', 3),  # class conv gradient, 20 classes
    (720, 80, True, 'd0_512', 2),         # class conv gradient, 80 classes
    (720, 80, False, 'wide_1024x512', 1),
    (64, None, False, 'd0_512', 3),       # a BiFPN node's output gradient
]


@pytest.mark.gpu
@pytest.mark.parametrize('C,width,prob,geo,B', TO_PLANES_CASES)
def test_to_planes(ops, C, width, prob, geo, B):
    """hi and lo bit for bit against bf16_rn(v), bf16_rn(v - hi) with v = x or (x * p) * (1 - p) computed by torch on the
    device; the pitch padding zero; the column sums of five level calls accumulated on a non-zero start"""
    levels = LEVEL_SETS[geo]
    g = _gen(C + B)
    pitch = ops._pitch8(C)
    stride = 256 // min(pitch // 8, 256)                 # rows a block of to_planes_kernel steps by
    assert stride == 2 or any(B * h * w % stride for h, w in levels)   # (every level has an even row count)
    if width is not None:
        offs, tot = _head_layout(levels, width)
        src = torch.full((B, tot, width), float('nan'), device=_dev())
        pr = torch.full((B, tot, width), float('nan'), device=_dev()) if prob else None
        xs, ps = [], []
        for (h, w), off in zip(levels, offs):
            v = _slice(src, off, h, w, width)
            v.copy_(_randn(g, B, h, w, C).to(_dev()))
            xs.append(v)
            if prob:
                p = _slice(pr, off, h, w, width)
                p.copy_(torch.sigmoid(_randn(g, B, h, w, C) * 3).to(_dev()))
                ps.append(p)
        ptrs = [(src.data_ptr() + 4 * off * width, tot * width) for off in offs]
        pptrs = [(pr.data_ptr() + 4 * off * width, tot * width) if prob else (None, 0) for off in offs]
    else:
        xs = [_randn(g, B, h, w, C).to(_dev()) for h, w in levels]
        ps = []
        ptrs = [(x.data_ptr(), h * w * C) for x, (h, w) in zip(xs, levels)]
        pptrs = [(None, 0)] * len(levels)
    assert max(B * h * w for h, w in levels) >= (1 << 20) or C != 36
    # fp64 column sums of every level, from the fp32 operands
    level_sums = []
    for i in range(len(levels)):
        xd = xs[i].double().cpu()
        if prob:
            pd = ps[i].double().cpu()
            xd = xd * pd * (1 - pd)
        level_sums.append(xd.sum(dim=(0, 1, 2)))
    # a non-zero start of the same order as the sums (a larger one would add its own fp32 rounding to the check)
    start = (_randn(g, C).double() * sum(level_sums).pow(2).mean().sqrt()).float()
    colsum = start.clone().to(_dev())
    planes = []
    for i, (h, w) in enumerate(levels):
        pl = _nan_planes(ops, B, h, w, C)
        ops.to_planes(ptrs[i][0], ptrs[i][1], pl, B, h * w, C, colsum, prob_ptr=pptrs[i][0], p_bs=pptrs[i][1], colsum=colsum)
        planes.append(pl)
    torch.cuda.synchronize()
    n_diff_order = 0
    for i, (h, w) in enumerate(levels):
        x = xs[i]
        v = (x * ps[i]) * (1 - ps[i]) if prob else x
        hi = v.to(torch.bfloat16)
        lo = (v - hi.float()).to(torch.bfloat16)
        pl = planes[i]
        assert torch.equal(_bits(pl[0, ..., :C]), _bits(hi)), ('hi', i)
        assert torch.equal(_bits(pl[1, ..., :C]), _bits(lo)), ('lo', i)
        if pitch > C:
            assert not _bits(pl[..., C:]).any(), ('pitch padding', i)
        if prob:
            # control: the other multiplication order gives other bits somewhere, so bit equality pins the order
            other = (x * (ps[i] * (1 - ps[i]))).to(torch.bfloat16)
            n_diff_order += int((_bits(other) != _bits(hi)).sum())
        else:
            # control: truncation instead of round-to-nearest gives other bits
            n_diff_order += int((_bits((x.contiguous().view(torch.int32) >> 16).to(torch.int16)) != _bits(hi)).sum())
    got_sum = colsum.cpu().double() - start.double()
    e = _rel(got_sum, sum(level_sums))
    miss = _rel(got_sum, sum(level_sums[1:]))            # control: a reference without level 0
    print('to_planes C=%d %s B=%d prob=%s: planes bit-exact; column sums rel err %.2e (bound %.0e), without level 0 %.2e; '
          '%d elements differ under the control rounding' % (C, geo, B, prob, e, TOL_SUM, miss, n_diff_order))
    assert e < TOL_SUM, e
    assert miss > TOL_SUM and n_diff_order > 0, (miss, n_diff_order)


@pytest.mark.gpu
def test_to_planes_refuses_channels_not_multiple_of_4(ops):
    x = torch.zeros(1, 4, 4, 812, device=_dev())
    pl = ops._planes(1, 4, 4, 810, x)
    with pytest.raises(ops.N.EffdetNativeError):
        ops.to_planes(x.data_ptr(), 16 * 810, pl, 1, 16, 810, x)


# ------------------------------------------------------------------------------------------------
# 3. conv_planes_kernel at the head's real launches
# ------------------------------------------------------------------------------------------------

def _mask_values(g, B, h, w, C):
    """what the forward stores as the ReLU output: about half exact +0, plus some -0.0 and positive subnormals (in the
    bf16 subnormal range: fp32 values below 2^-134 round to +0 in both planes, so the planes cannot hold them)"""
    m = torch.relu(_randn(g, B, h, w, C))
    sel = torch.rand(m.shape, generator=g)
    m[sel < 0.02] = -0.0
    m[(sel >= 0.02) & (sel < 0.03)] = 1e-39
    m[(sel >= 0.03) & (sel < 0.04)] = 5e-40
    return m


@pytest.mark.gpu
@pytest.mark.parametrize('Co', [36, 180, 720])
@pytest.mark.parametrize('geo,B', [('d0_512', 2), ('wide_1024x512', 1)])
def test_head_output_conv(ops, Co, geo, B):
    """forward of the box (F -> 36, no activation) or class conv (F -> 9K, sigmoid) into slices of one concatenated
    [B, tot, width] output (y_bs = tot*width); then the data gradient 9K / 36 -> F from planes of a strided source,
    with ReLU mask planes and column sums"""
    levels = LEVEL_SETS[geo]
    Fw = 64
    width = Co // A
    act = ops.ACT_NONE if Co == 36 else ops.ACT_SIGMOID
    g = _gen(Co * 7 + B)
    xs = [_randn(g, B, h, w, Fw) for h, w in levels]
    w = _randn(g, Co, Fw, 3, 3) * (1.0 / (9 * Fw) ** 0.5)
    bias = _randn(g, Co) * 0.1
    wd, bd = w.to(_dev()), bias.to(_dev())
    fwd, dgr = ops.tc_packs(wd)
    xp = [_to_planes(ops, x.to(_dev())) for x in xs]
    offs, tot = _head_layout(levels, width)
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    conv = [_nhwc(F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), bias.double(), 1, 1)) for x in xs]

    out = torch.full((B, tot, width), float('nan'), device=_dev())
    ops.conv_planes_multi(out, [dict(x=xp[i], y_ptr=out.data_ptr() + 4 * offs[i] * width, y_bs=tot * width, B=B, H=h, W=w_)
                                for i, (h, w_) in enumerate(levels)], fwd, Fw, Co, 3, bias=bd, act=act)
    f = torch.sigmoid if act == ops.ACT_SIGMOID else (lambda t: t)
    outc = out.cpu()
    got = [_slice(outc, off, h, w_, width) for off, (h, w_) in zip(offs, levels)]
    _check(got, [f(c) for c in conv], 'head %s 64->%d forward %s B=%d' % ('sigmoid' if Co != 36 else 'linear', Co, geo, B))
    written = torch.zeros(tot, dtype=torch.bool)
    for off, (h, w_) in zip(offs, levels):
        written[off:off + h * w_ * A] = True
    assert torch.isnan(outc[:, ~written]).all() and not torch.isnan(outc[:, written]).any()
    # control: one bf16 product per multiply-add, same launch without the activation
    lin = torch.full((B, tot, width), float('nan'), device=_dev())
    with _single_pass(ops):
        ops.conv_planes_multi(lin, [dict(x=xp[i], y_ptr=lin.data_ptr() + 4 * offs[i] * width, y_bs=tot * width, B=B, H=h, W=w_)
                                    for i, (h, w_) in enumerate(levels)], fwd, Fw, Co, 3, bias=bd)
    lin = lin.cpu()
    single = _rel(torch.cat([_slice(lin, o, h, w_, width).flatten() for o, (h, w_) in zip(offs, levels)]),
                  torch.cat([c.flatten() for c in conv]))
    assert single > SINGLE_PASS_MIN, single

    # data gradient: planes of the strided head-output gradient (GEMM-K = Co, pitch padded to 8 when Co % 8 == 4)
    dsrc = torch.full((B, tot, width), float('nan'), device=_dev())
    dys = []
    for off, (h, w_) in zip(offs, levels):
        d = _randn(g, B, h, w_, Co)
        _slice(dsrc, off, h, w_, width).copy_(d.to(_dev()))
        dys.append(d)
    dp = []
    for off, (h, w_) in zip(offs, levels):
        pl = ops._planes(B, h, w_, Co, dsrc)
        ops.to_planes(dsrc.data_ptr() + 4 * off * width, tot * width, pl, B, h * w_, Co, dsrc)
        dp.append(pl)
    ms = [_mask_values(g, B, h, w_, Fw) for h, w_ in levels]
    mp = [_to_planes(ops, m.to(_dev())) for m in ms]
    start = _randn(g, Fw) * 10.0
    colsum = start.clone().to(_dev())
    dx = [_nan_planes(ops, B, h, w_, Fw) for h, w_ in levels]

    def dgrad(ys, cs):
        ops.conv_planes_multi(dsrc, [dict(x=dp[i], y_planes=ys[i], mask=mp[i], B=B, H=h, W=w_) for i, (h, w_) in enumerate(levels)],
                              dgr, Co, Fw, 3, colsum=cs)

    dgrad(dx, colsum)
    tr = [_nhwc(F.conv_transpose2d(d.permute(0, 3, 1, 2).double(), w.double(), None, 1, 1)) for d in dys]
    want = [t * (m > 0) for t, m in zip(tr, ms)]
    got = [_from_planes(p, Fw) for p in dx]
    _check(got, want, 'head %d->64 data gradient, ReLU mask %s B=%d' % (Co, geo, B))
    e = _rel(colsum.cpu().double() - start.double(), sum(t.sum(dim=(0, 1, 2)) for t in want))
    print('  column sums rel err %.2e (bound %.0e)' % (e, TOL_TC))
    assert e < TOL_TC, e
    # controls: a mask that passes +0 / -0, and one bf16 product per multiply-add
    zero_pos = _rel(torch.cat([t.flatten() for t in got]), torch.cat([(t * (m >= 0)).flatten() for t, m in zip(tr, ms)]))
    dx1 = [_nan_planes(ops, B, h, w_, Fw) for h, w_ in levels]
    with _single_pass(ops):
        dgrad(dx1, None)
    single = _rel(torch.cat([_from_planes(p, Fw).flatten() for p in dx1]), torch.cat([t.flatten() for t in want]))
    print('  controls: zeros passed %.2e, single pass %.2e' % (zero_pos, single))
    assert zero_pos > 1e-2 and single > SINGLE_PASS_MIN, (zero_pos, single)


@pytest.mark.gpu
@pytest.mark.parametrize('residual', [False, True])
def test_head_first_layer_data_gradient(ops, residual):
    """the data gradient of each tower's first conv, F -> Cin into fp32: the class tower writes it, the box tower adds
    the class tower's result (res_ptr)"""
    levels = LEVEL_SETS['d0_512']
    B, Fw, Cin = 2, 64, 64
    g = _gen(11 + residual)
    ds = [_randn(g, B, h, w, Fw) for h, w in levels]
    res = [_randn(g, B, h, w, Cin) for h, w in levels]
    w = _randn(g, Fw, Cin, 3, 3) * (1.0 / (9 * Fw) ** 0.5)           # the layer Cin -> F
    wd = w.to(_dev())
    _, dgr = ops.tc_packs(wd)
    dp = [_to_planes(ops, d.to(_dev())) for d in ds]
    resd = [r.to(_dev()) for r in res]

    def launch():
        out = [torch.full((B, h, w_, Cin), float('nan'), device=_dev()) for h, w_ in levels]
        ops.conv_planes_multi(wd, [dict(x=dp[i], y_ptr=out[i].data_ptr(), y_bs=h * w_ * Cin,
                                        res_ptr=resd[i].data_ptr() if residual else None, res_bs=h * w_ * Cin, B=B, H=h, W=w_)
                                   for i, (h, w_) in enumerate(levels)], dgr, Fw, Cin, 3)
        return [o.double().cpu() for o in out]

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    want = [_nhwc(F.conv_transpose2d(d.permute(0, 3, 1, 2).double(), w.double(), None, 1, 1)) + (r.double() if residual else 0)
            for d, r in zip(ds, res)]
    _check(launch(), want, 'tower first layer data gradient%s' % (' + residual' if residual else ''))
    with _single_pass(ops):
        got = launch()
    # control against the convolution alone (the residual would dilute the single-pass error)
    single = _rel(torch.cat([(o - (r.double() if residual else 0)).flatten() for o, r in zip(got, res)]),
                  torch.cat([(t - (r.double() if residual else 0)).flatten() for t, r in zip(want, res)]))
    assert single > SINGLE_PASS_MIN, single


# ------------------------------------------------------------------------------------------------
# 4. BiFPN fusion kernels
# ------------------------------------------------------------------------------------------------

EPS = 1e-4
# raw fusion weights of the node's column: small positive weights make the eps terms of both normalisations visible
# (without eps the normalisation is scale invariant); the other sets hold a negative and an exactly-zero weight,
# whose gradient must be exactly 0
WEIGHT_SETS = {2: [[0.006, 0.011], [-0.4, 0.011], [0.0, 0.011]],
               3: [[0.006, 0.011, 0.004], [-0.4, 0.011, 0.004], [0.006, 0.0, 0.004]]}
ACC_FLAGS = [(0, 0, 0), (1, 1, 1), (1, 0, 1)]
SHAPES = {'square': (32, 32), 'wide': (48, 80)}          # the UP node's fine grid; a POOL node's output is half of it


def _resample(b, mode, ops):
    if mode == ops.FUSE_UP:
        return b.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    return _nhwc(F.max_pool2d(b.permute(0, 3, 1, 2), 2, 2))


def _fuse_ref(ins, wcol, mode, ops, detach_second=False):
    r = torch.relu(wcol)
    n = r / (r.sum() + EPS)
    s = n[0] * ins[0] + n[1] * _resample(ins[1], mode, ops)
    if len(ins) == 3:
        s = s + n[2] * ins[2]
    D = n.sum() + EPS
    return s / (D.detach() if detach_second else D)


def _pool_last_max(b, gb):
    """the max-pool backward routed to the LAST maximum of each window (the wrong tie rule)"""
    B_, H2, W2, C = b.shape
    win = b.reshape(B_, H2 // 2, 2, W2 // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B_, H2 // 2, W2 // 2, C, 4)
    idx = 3 - win.flip(-1).argmax(dim=-1)                  # argmax returns the first; flipped -> the last
    out = torch.zeros_like(win)
    out.scatter_(-1, idx.unsqueeze(-1), gb.unsqueeze(-1))
    return out.reshape(B_, H2 // 2, W2 // 2, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B_, H2, W2, C)


def _fusion_case(ops, mode, nin, C, B, H, W, seed, weight_sets, acc_flags, check_values=True):
    """forward (fp32 and planes) and backward of one fusion node for each raw weight set; returns the worst errors"""
    g = _gen(seed)
    bshape = (B, H // 2, W // 2, C) if mode == ops.FUSE_UP else (B, 2 * H, 2 * W, C)
    a = _randn(g, B, H, W, C)
    b = _randn(g, *bshape)
    if mode == ops.FUSE_POOL:
        b = torch.round(b * 2) / 2                        # coarse values: most 2x2 windows hold exact ties
    c = _randn(g, B, H, W, C) if nin == 3 else None
    dout = _randn(g, B, H, W, C)
    ad, bd_, cd, doutd = a.to(_dev()), b.to(_dev()), c.to(_dev()) if c is not None else None, dout.to(_dev())
    ins64 = [t.double() for t in (a, b, c) if t is not None]
    worst = dict(fwd=0.0, planes=0, data=0.0, dw=0.0, ctrl_dw=float('inf'), ctrl_tie=float('inf'))
    col, L = 1, 3
    for k, ws in enumerate(weight_sets):
        wm = torch.rand(nin, L, generator=g) + 0.1
        wm[:, col] = torch.tensor(ws)
        wmd = wm.to(_dev())
        wcol = torch.tensor(ws, dtype=torch.float64, requires_grad=True)
        leaves = [t.clone().requires_grad_(True) for t in ins64]
        ref = _fuse_ref(leaves, wcol, mode, ops)
        # forward: fp32 output, and the planes output bit for bit against it
        out = ops._fuse_fwd(ad, bd_, cd, wmd, col, EPS, mode)
        pl = ops._fuse_fwd(ad, bd_, cd, wmd, col, EPS, mode, planes=True)
        e = _rel(out, ref.detach())
        worst['fwd'] = max(worst['fwd'], e)
        assert e < TOL_EXACT, ('forward', k, e)
        hi = out.to(torch.bfloat16)
        lo = (out - hi.float()).to(torch.bfloat16)
        assert torch.equal(_bits(pl[0]), _bits(hi)) and torch.equal(_bits(pl[1]), _bits(lo)), ('planes', k)
        # backward: NaN where the kernel writes, random values where it adds
        ref.backward(dout.double())
        acc = acc_flags[k]
        bufs, starts = [], []
        for t, f in zip((a, b, c), acc):
            if t is None:
                bufs.append(None)
                starts.append(None)
                continue
            s0 = _randn(g, *t.shape) if f else torch.full(t.shape, float('nan'))
            starts.append(s0)
            bufs.append(s0.to(_dev()))
        dw0 = _randn(g, nin, L) * 0.1
        dwd = dw0.to(_dev())
        ops._fuse_bwd(doutd, ad, bd_, cd, wmd, col, EPS, mode, bufs[0], acc[0], bufs[1], acc[1], bufs[2], acc[2], dwd)
        for j, (buf, s0, f, leaf) in enumerate(zip(bufs, starts, acc, leaves + [None])):
            if buf is None or leaf is None:
                continue
            want = leaf.grad + (s0.double() if f else 0)
            e = _rel(buf, want)
            worst['data'] = max(worst['data'], e)
            assert e < TOL_EXACT, ('data gradient', 'abc'[j], k, e)
        if mode == ops.FUSE_POOL and k == 0:
            # control: routing ties to the last maximum of the window gives another db
            alt = _pool_last_max(ins64[1], _pooled_grad(wcol, dout.double()))
            worst['ctrl_tie'] = min(worst['ctrl_tie'], _rel(bufs[1].double().cpu() - (starts[1].double() if acc[1] else 0), alt))
        dw = dwd.cpu()
        others = [j for j in range(L) if j != col]
        assert torch.equal(dw[:, others], dw0[:, others]), 'columns of other nodes changed'
        active = [j for j in range(nin) if ws[j] > 0]
        for j in range(nin):
            if ws[j] <= 0:
                assert dw[j, col] == dw0[j, col], ('gradient of a clamped weight', ws, j)
        if len(active) >= 2:
            # with one active weight its gradient is eps/(r+eps) of two nearly equal fp32 terms: not checked
            got = dw[active, col].double() - dw0[active, col].double()
            # the gradient is a difference of terms of size |T| / (D E) (dn_j = T_j / D - nT / D^2, T_j = sum(dout * in_j)):
            # where the T_j are close it cancels, and its fp32 error is measured against the size of those terms
            res = [ins64[0], _resample(ins64[1], mode, ops)] + ins64[2:]
            T = torch.stack([(dout.double() * t).sum() for t in res])
            r = torch.relu(torch.tensor(ws, dtype=torch.float64))
            E = r.sum() + EPS
            D = (r / E).sum() + EPS
            want = wcol.grad[active]

            def err(x):
                return float((x - want).norm()) / max(float(want.norm()), float(T.norm() / (D * E)))

            e = err(got)
            worst['dw'] = max(worst['dw'], e)
            assert e < TOL_SUM, ('weight gradient', ws, e)
            if len(active) == nin:
                # control: the same metric for a gradient without the second normalisation's term (D held constant)
                wc2 = torch.tensor(ws, dtype=torch.float64, requires_grad=True)
                (_fuse_ref([t.detach() for t in ins64], wc2, mode, ops, detach_second=True) * dout.double()).sum().backward()
                worst['ctrl_dw'] = min(worst['ctrl_dw'], err(wc2.grad[active]))
    return worst


def _pooled_grad(wcol, dout):
    """the gradient that arrives at the pooled map: dout * n1 / D"""
    r = torch.relu(wcol.detach())
    n = r / (r.sum() + EPS)
    return dout * (n[1] / (n.sum() + EPS))


@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('C', [64, 88, 384])
@pytest.mark.parametrize('nin', [2, 3])
@pytest.mark.parametrize('mode', ['up', 'pool'])
def test_bifpn_fusion(ops, mode, nin, C, shape, B):
    """fuse_fwd_kernel (fp32 and planes output) and fuse_bwd_{up,pool}_kernel + fuse_bwd_weights_kernel against fp64
    autograd through both normalisations, with the accumulate flags, max-pool ties and clamped weights"""
    m = ops.FUSE_UP if mode == 'up' else ops.FUSE_POOL
    H, W = SHAPES[shape]
    if m == ops.FUSE_POOL:
        H, W = H // 2, W // 2
    w = _fusion_case(ops, m, nin, C, B, H, W, seed=C * 10 + B + nin * 1000 + (mode == 'up') * 5000 + H,
                     weight_sets=WEIGHT_SETS[nin], acc_flags=ACC_FLAGS)
    print('fusion %s nin=%d C=%d %dx%d B=%d: fwd %.2e, data %.2e (bound %.0e), weights %.2e (bound %.0e); controls: '
          'without the second normalisation %.2e, ties to the last maximum %.2e'
          % (mode, nin, C, H, W, B, w['fwd'], w['data'], TOL_EXACT, w['dw'], TOL_SUM, w['ctrl_dw'], w['ctrl_tie']))
    assert w['ctrl_dw'] > 2 * TOL_SUM, w['ctrl_dw']
    if m == ops.FUSE_POOL:
        assert w['ctrl_tie'] > 10 * TOL_EXACT, w['ctrl_tie']


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['up', 'pool'])
def test_bifpn_fusion_weight_gradient_many_blocks(ops, mode):
    """a 128x128 (pool) / 256x256 (up) node at B=4: the fusion-weight gradient's partial sums come from 4096 blocks"""
    m = ops.FUSE_UP if mode == 'up' else ops.FUSE_POOL
    H = W = 256 if m == ops.FUSE_UP else 128
    B, C = 4, 64
    blocks = _cdiv(B * (H // 2 if m == ops.FUSE_UP else H) * (W // 2 if m == ops.FUSE_UP else W) * C // 4, 256)
    assert blocks >= 4096
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    w = _fusion_case(ops, m, 3, C, B, H, W, seed=77 + (mode == 'up'), weight_sets=WEIGHT_SETS[3][:1], acc_flags=ACC_FLAGS[:1])
    print('fusion %s %dx%d B=%d, %d blocks: weights %.2e (bound %.0e), without the second normalisation %.2e'
          % (mode, H, W, B, blocks, w['dw'], TOL_SUM, w['ctrl_dw']))
    assert w['ctrl_dw'] > 2 * TOL_SUM, w['ctrl_dw']
