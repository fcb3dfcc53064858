"""conv_planes_kernel's epilogue: the one-bit ReLU mask a forward writes (y_mask) and a data gradient reads
(mask_bits), and the per-CTA column sums.

  forward   a ReLU forward into planes also writes y_mask: bit c % 32 of word (pixel, c // 32) is set exactly when the
            stored bf16 pair (hi, lo) of channel c is > 0, i.e. (hi & 0x7fff) ? !(hi & 0x8000) : (lo & 0x7fff) &&
            !(lo & 0x8000).  Every word of every valid pixel is written (a partial last word has its unused bits
            clear), nothing past the last pixel is.
  dgrad     the data gradient with mask_bits stores the same planes, bit for bit, as with the forward's planes as the
            mask (mask=), and both equal the float64 reference; the column sums (bias gradient) do too.

Shapes: the benchmark's tower layer (B = 32, P3..P7 of 512^2, 256 channels: 2728 units of 128 x 128 over 132 CTAs,
so 20 or 21 per CTA and the second consumer warpgroup runs one unit fewer in some CTAs), the box conv's data gradient
36 -> 256 at the same levels, D4's 224 channels (7 words per pixel) and 40 channels (a partial last word) at a
batch small enough that every CTA has one unit and the second warpgroup idles.  Bounds as in test_planes_path_parity:
TOL_TC / TOL_LOCAL for the gradient planes, TOL_SUM for the column sums; the float64 references run on the device."""
import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O

TOL_TC = 3e-5
TOL_LOCAL = 1e-4
TOL_SUM = 2e-5
D0_512 = [(64, 64), (32, 32), (16, 16), (8, 8), (4, 4)]
GUARD = 64                      # words past each y_mask that the forward must leave alone


def _dev():
    return torch.device('cuda:0')


@pytest.fixture(params=['bf16x3', 'bf16'])
def ops(request):
    from models import _ops
    old = _ops.PRECISION
    _ops.PRECISION = request.param
    yield _ops
    _ops.PRECISION = old


def _to_planes(ops, x):
    b, h, w, c = x.shape
    p = ops._planes(b, h, w, c, x)
    ops.to_planes(x.data_ptr(), h * w * c, p, b, h * w, c, x)
    return p


def _bits_of_planes(p, C):
    """the ReLU predicate of planes [2, B, H, W, pitch] on their raw bf16 bits, packed as y_mask words"""
    hb = p[0, ..., :C].view(torch.int16).int() & 0xffff
    lb = p[1, ..., :C].view(torch.int16).int() & 0xffff
    pos = torch.where((hb & 0x7fff) != 0, (hb & 0x8000) == 0, ((lb & 0x7fff) != 0) & ((lb & 0x8000) == 0))
    nw = (C + 31) // 32
    pos = F.pad(pos, (0, nw * 32 - C)).reshape(*pos.shape[:-1], nw, 32).long()
    words = (pos << torch.arange(32, device=pos.device)).sum(-1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).int()


def _relu_forward(ops, g, B, levels, Cin, Cout):
    """a ReLU forward Cin -> Cout into planes and y_mask; the masks sit in front of a guard of GUARD sentinel words"""
    xs = [_to_planes(ops, torch.randn(B, h, w, Cin, device=_dev(), generator=g)) for h, w in levels]
    wt = torch.randn(Cout, Cin, 3, 3, device=_dev(), generator=g) / (9 * Cin) ** 0.5
    bias = torch.randn(Cout, device=_dev(), generator=g) * 0.1
    nw = (Cout + 31) // 32
    ys = [ops._planes(B, h, w, Cout, xs[0]) for h, w in levels]
    store = [torch.full((B * h * w * nw + GUARD,), 0x5a5a5a5a, device=_dev(), dtype=torch.int32) for h, w in levels]
    bits = [s[:B * h * w * nw].view(B, h, w, nw) for s, (h, w) in zip(store, levels)]
    ops.conv_planes_multi(wt, [dict(x=xs[i], y_planes=ys[i], y_mask=bits[i], B=B, H=h, W=w) for i, (h, w) in enumerate(levels)],
                          ops.tc_packs(wt)[0], Cin, Cout, 3, bias=bias, act=ops.ACT_RELU)
    return ys, bits, store


@pytest.mark.gpu
@pytest.mark.parametrize('Cin,Cout,B', [(256, 256, 32), (64, 256, 32), (224, 224, 3), (64, 40, 3)])
def test_forward_writes_relu_bits_of_its_planes(ops, Cin, Cout, B):
    g = torch.Generator(device=_dev()).manual_seed(Cout * 100 + B)
    ys, bits, store = _relu_forward(ops, g, B, D0_512, Cin, Cout)
    for i, (y, b, s) in enumerate(zip(ys, bits, store)):
        want = _bits_of_planes(y, Cout)
        assert torch.equal(b, want), ('level', i, int((b != want).sum()))
        assert (s[-GUARD:] == 0x5a5a5a5a).all(), ('written past the last pixel', i)
        if Cout % 32:
            assert not (b[..., -1] >> (Cout % 32)).any(), ('bits past the last channel', i)
        frac = float(torch.cat([((y[0, ..., :Cout].float() + y[1, ..., :Cout].float()) > 0).flatten()]).float().mean())
        assert 0.2 < frac < 0.8, frac                   # both halves of the predicate occur


@pytest.mark.gpu
@pytest.mark.parametrize('Co,Fw,B', [(256, 256, 32), (36, 256, 32), (224, 224, 3), (40, 40, 3)])
def test_masked_data_gradient_from_bits(ops, Co, Fw, B):
    """the data gradient Co -> Fw of a layer whose input is a ReLU forward's output: mask_bits and mask= planes give
    the same planes, and the float64 reference (bf16x3) within the parity bounds, column sums included"""
    levels = D0_512
    g = torch.Generator(device=_dev()).manual_seed(Co * 1000 + Fw + B)
    ms, bits, _ = _relu_forward(ops, g, B, levels, 64, Fw)
    dys = [torch.randn(B, h, w, Co, device=_dev(), generator=g) for h, w in levels]
    dp = [_to_planes(ops, d) for d in dys]
    wt = torch.randn(Co, Fw, 3, 3, device=_dev(), generator=g) / (9 * Fw) ** 0.5
    dgr = ops.tc_packs(wt)[1]
    start = torch.randn(Fw, device=_dev(), generator=g) * 10.0

    def dgrad(mask_key, masks):
        dx = [torch.full((2, B, h, w, ops._pitch8(Fw)), float('nan'), device=_dev(), dtype=torch.bfloat16) for h, w in levels]
        cs = start.clone()
        ops.conv_planes_multi(wt, [{'x': dp[i], 'y_planes': dx[i], mask_key: masks[i], 'B': B, 'H': h, 'W': w}
                                   for i, (h, w) in enumerate(levels)], dgr, Co, Fw, 3, colsum=cs)
        return dx, cs

    dx_bits, cs_bits = dgrad('mask_bits', bits)
    dx_planes, cs_planes = dgrad('mask', ms)
    for i in range(len(levels)):
        assert torch.equal(dx_bits[i][..., :Fw].view(torch.int16), dx_planes[i][..., :Fw].view(torch.int16)), ('level', i)
    assert O.rel_err(cs_bits.double() - start.double(), cs_planes.double() - start.double()) < TOL_SUM
    if ops.PRECISION != 'bf16x3':
        return
    want = []
    for d, m in zip(dys, ms):
        t = F.conv_transpose2d(d.permute(0, 3, 1, 2).double(), wt.double(), None, 1, 1).permute(0, 2, 3, 1)
        want.append(t * ((m[0, ..., :Fw].double() + m[1, ..., :Fw].double()) > 0))
    got = [(p[0].double() + p[1].double())[..., :Fw] for p in dx_bits]
    e = O.rel_err(torch.cat([t.flatten() for t in got]).cpu(), torch.cat([t.flatten() for t in want]).cpu())
    loc = max(O.rel_err(a.cpu(), b.cpu()) for a, b in zip(got, want))
    es = O.rel_err((cs_bits.double() - start.double()).cpu(), sum(t.sum(dim=(0, 1, 2)) for t in want).cpu())
    print('%d->%d B=%d: rel err %.2e, worst level %.2e, column sums %.2e' % (Co, Fw, B, e, loc, es))
    assert e < TOL_TC and loc < TOL_LOCAL, (e, loc)
    assert es < TOL_SUM, es


def test_mask_arguments_are_validated():
    """both mask sources in one call, a y_mask on a launch without ReLU planes, and column sums wider than shared
    memory are refused before anything touches the device"""
    from models import _native as N
    lib = N.load()
    fake = 1 << 20

    def call(**kw):
        a = dict(x_planes=fake, w_tc=fake, y_planes=fake, B=1, H=8, W=8, Cin=64, Cout=64, ksize=3, act=1)
        a.update(kw)
        arr = (N.ConvPlanesArgs * 1)(N.ConvPlanesArgs(**a))
        return lib.effdet_conv_planes_multi(arr, 1, 0, None), lib.effdet_last_error().decode()

    rc, err = call(mask_planes=fake, mask_bits=fake)
    assert rc != 0 and 'both' in err, err
    rc, err = call(y_mask=fake, act=0)
    assert rc != 0 and 'y_mask' in err, err
    rc, err = call(y_mask=fake, y_planes=None, y=fake)
    assert rc != 0 and 'y_mask' in err, err
    rc, err = call(Cout=4096, colsum=fake)
    assert rc != 0 and 'shared memory' in err, err
