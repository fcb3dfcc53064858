"""conv_planes_kernel's ping-pong schedule: a CTA's k-th unit belongs to consumer warpgroup k & 1, the two take turns
on the stage ring, and one warpgroup's epilogue runs under the other's MMAs.  The geometries here are sized from the
device's SM count so that the CTAs run 1, 2, 3 or 5 units (one warpgroup only, one hand-over, a second turn of
warpgroup 0, an odd count with both warpgroups turning twice), over a mix of pyramid levels, for both tile widths
(Cout <= 64: 64 columns, else 128, with a partial last channel tile at 720) in both precision modes.  Every epilogue
feature is checked against fp64 F.conv2d / conv_transpose2d: bias + ReLU -> planes, sigmoid -> fp32, residual,
ReLU mask + column sums."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'tools'))
import bf16_emulation as E  # noqa: E402

pytestmark = pytest.mark.gpu

TOL_TC = 3e-5                       # the kernel tests' bound: fp32 accumulation of (split) bf16 products
LEVELS = [(16, 16), (8, 8), (4, 4)]


def _dev():
    return torch.device('cuda:0')


@pytest.fixture(params=['bf16x3', 'bf16'])
def ops(request):
    from models import _ops
    old = _ops.PRECISION
    _ops.PRECISION = request.param
    yield _ops
    _ops.PRECISION = old


def _tiles(B, H, W):
    """128-row pixel tiles of one level (the pixel box of wg_geometry, conv_tc.cu)"""
    Wb = min(W, 64)
    Hb = max(h for h in range(1, H + 1) if H % h == 0 and Wb * h <= 64)
    Bb = min(max(64 // (Wb * Hb), 1), B)
    ks = Wb * Hb * Bb
    boxes = (W // Wb) * (H // Hb) * -(-B // Bb)
    return -(-boxes // (128 // ks))


def _busiest_cta(B, ntn, sms):
    """units of the busiest CTA (the grid is min(units, SMs))"""
    units = sum(_tiles(B, h, w) for h, w in LEVELS) * ntn
    return -(-units // min(units, sms))


def _batch(units_per_cta, Cout):
    """the largest batch whose busiest CTAs run units_per_cta units"""
    sms = torch.cuda.get_device_properties(_dev()).multi_processor_count
    ntn = -(-Cout // (64 if Cout <= 64 else 128))
    B = max(b for b in range(1, 1024) if _busiest_cta(b, ntn, sms) <= units_per_cta)
    assert _busiest_cta(B, ntn, sms) == units_per_cta, (units_per_cta, Cout)
    return B


def _planes(ops, ts, C):
    out = []
    for t in ts:
        b, h, w, _ = t.shape
        p = ops._planes(b, h, w, C, t)
        ops.to_planes(t.data_ptr(), h * w * C, p, b, h * w, C, t)
        out.append(p)
    return out


def _from_planes(p, C):
    return (p[0].double() + p[1].double())[..., :C]


def _check(ops, got, want, what):
    e = O.rel_err(torch.cat([t.flatten() for t in got]), torch.cat([t.flatten() for t in want]))
    print(what, ops.PRECISION, 'rel err %.2e' % e)
    assert e < TOL_TC, (what, ops.PRECISION, e)


def _ref(ops, x, w):
    """fp64 operands as the kernel multiplies them: hi + lo (bf16x3, ~ the fp32 value) or hi alone (bf16)"""
    r = E.rn if ops.PRECISION == 'bf16' else (lambda t: t)
    return r(x).double(), r(w).double()


@pytest.mark.parametrize('units_per_cta', [1, 2, 3, 5])
@pytest.mark.parametrize('Cin,Cout', [(64, 64), (256, 720)])
def test_planes_schedule_forward(ops, Cin, Cout, units_per_cta):
    B = _batch(units_per_cta, Cout)
    g = torch.Generator(device=_dev()).manual_seed(1000 * units_per_cta + Cout)
    xs = [torch.randn(B, h, w, Cin, device=_dev(), generator=g) for h, w in LEVELS]
    res = [torch.randn(B, h, w, Cout, device=_dev(), generator=g) for h, w in LEVELS]
    w = torch.randn(Cout, Cin, 3, 3, device=_dev(), generator=g) * (1.0 / (9 * Cin) ** 0.5)
    bias = torch.randn(Cout, device=_dev(), generator=g) * 0.1
    fwd, _ = ops.tc_packs(w)
    xp = _planes(ops, xs, Cin)
    conv = []
    for x in xs:
        xd, wd = _ref(ops, x.permute(0, 3, 1, 2), w)
        conv.append((F.conv2d(xd, wd, None, 1, 1) + bias.double().view(1, -1, 1, 1)).permute(0, 2, 3, 1))

    def launch(act, **kw):
        ops.conv_planes_multi(w, [dict(x=xp[i], B=B, H=h, W=wd, **{k: v[i] for k, v in kw.items()})
                                  for i, (h, wd) in enumerate(LEVELS)], fwd, Cin, Cout, 3, bias=bias, act=act)

    ys = [ops._planes(B, h, w_, Cout, x) for (h, w_), x in zip(LEVELS, xs)]
    launch(ops.ACT_RELU, y_planes=ys)
    _check(ops, [_from_planes(y, Cout) for y in ys], [torch.relu(c) for c in conv], 'bias + ReLU -> planes')

    yf = [torch.empty(B, h, w_, Cout, device=_dev()) for h, w_ in LEVELS]
    launch(ops.ACT_SIGMOID, y_ptr=[y.data_ptr() for y in yf], y_bs=[h * w_ * Cout for h, w_ in LEVELS])
    _check(ops, yf, [torch.sigmoid(c) for c in conv], 'sigmoid -> fp32')

    yf = [torch.empty(B, h, w_, Cout, device=_dev()) for h, w_ in LEVELS]
    launch(ops.ACT_NONE, y_ptr=[y.data_ptr() for y in yf], y_bs=[h * w_ * Cout for h, w_ in LEVELS],
           res_ptr=[r.data_ptr() for r in res], res_bs=[h * w_ * Cout for h, w_ in LEVELS])
    _check(ops, yf, [c + r.double() for c, r in zip(conv, res)], 'bias + residual -> fp32')


@pytest.mark.parametrize('units_per_cta', [1, 2, 3, 5])
@pytest.mark.parametrize('Cin,Cout', [(64, 64), (720, 256)])
def test_planes_schedule_data_gradient(ops, Cin, Cout, units_per_cta):
    """the data gradient of a Cout -> Cin layer (a Cin -> Cout launch on the dgrad pack): ReLU mask of the layer input
    from its planes, column sums of what is stored (the bias gradient of the layer below)"""
    B = _batch(units_per_cta, Cout)
    g = torch.Generator(device=_dev()).manual_seed(2000 * units_per_cta + Cin)
    dys = [torch.randn(B, h, w, Cin, device=_dev(), generator=g) for h, w in LEVELS]
    ms = [torch.randn(B, h, w, Cout, device=_dev(), generator=g) for h, w in LEVELS]
    w = torch.randn(Cin, Cout, 3, 3, device=_dev(), generator=g) * (1.0 / (9 * Cin) ** 0.5)   # the layer's Cout -> Cin
    _, dgr = ops.tc_packs(w)
    dyp, mp = _planes(ops, dys, Cin), _planes(ops, ms, Cout)
    dxs = [ops._planes(B, h, w_, Cout, d) for (h, w_), d in zip(LEVELS, dys)]
    colsum = torch.zeros(Cout, device=_dev())
    ops.conv_planes_multi(w, [dict(x=dyp[i], y_planes=dxs[i], mask=mp[i], B=B, H=h, W=w_) for i, (h, w_) in enumerate(LEVELS)],
                          dgr, Cin, Cout, 3, colsum=colsum)
    want = []
    for d, m in zip(dys, ms):
        dd, wd = _ref(ops, d.permute(0, 3, 1, 2), w)
        want.append(F.conv_transpose2d(dd, wd, None, 1, 1).permute(0, 2, 3, 1) * (m > 0))
    _check(ops, [_from_planes(d, Cout) for d in dxs], want, 'ReLU mask -> planes')
    _check(ops, [colsum], [sum(t.sum(dim=(0, 1, 2)) for t in want)], 'column sums')
