"""The tensor-core weight gradients' tap-major accumulation: wgrad_tc2_multi_kernel and wgrad_tc_kernel add their
partial sums into an fp32 [taps][Cout][Cin] accumulator with 16-byte vector reductions.  For a 3x3 conv that is the
ws_dw workspace, which the router clears before the launches and wgrad_fold_kernel adds into the OIHW dw after them;
for a 1x1 conv [1][Cout][Cin] is OIHW itself, so the kernels reduce straight into dw.

  * fp64 parity at the benchmarked step's launch plans (D0 512^2, B = 32, P3..P7 in one launch) for every 3x3 weight
    gradient class of the step, in bf16x3 and in bf16 mode, added onto a non-zero dw;
  * a 1x1 weight gradient with a bias gradient (not the pointwise kernel's job): TMA-fed and gathering routes, into dw;
  * a 3x3 call with one level on each tensor-core route (the 2x2 map has no pixel box), one fold for both;
  * the refusal of a 3x3 tensor-core call without ws_dw, before any device work.

Bounds as in test_planes_path_parity.py: TOL_TC on the whole tensor, TOL_LOCAL on every block of 64 output channels x
tap.  In bf16 mode the kernels multiply the bf16 hi halves of the operands once each, with fp32 accumulation, so the
reference there is built from those hi halves and the same bounds apply."""
import ctypes

import pytest
import torch

import effdet_oracle as O

TOL_TC = 3e-5
TOL_LOCAL = 1e-4
D0_512 = [(64, 64), (32, 32), (16, 16), (8, 8), (4, 4)]
# (Cin, Cout) of the 3x3 weight gradients of the D0 train step: tower, class conv (80 classes), box conv, first tower
# layer (BiFPN width 64), BiFPN node conv
BENCH_PAIRS = [(256, 256), (256, 720), (256, 36), (64, 256), (64, 64)]


@pytest.fixture()
def ops():
    from models import _ops
    old = _ops.PRECISION
    yield _ops
    _ops.PRECISION = old


def _dev():
    return torch.device('cuda:0')


def _planes(ops, x):
    b, h, w, c = x.shape
    p = ops._planes(b, h, w, c, x)
    ops.to_planes(x.data_ptr(), h * w * c, p, b, h * w, c, x)
    return p


def _ref(xs, dys, k):
    """fp64 weight gradient summed over levels, OIHW, on the device; xs / dys: NHWC"""
    Cin, Cout = xs[0].shape[3], dys[0].shape[3]
    return sum(torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2).double(), (Cout, Cin, k, k),
                                           d.permute(0, 3, 1, 2).double(), 1, k // 2) for x, d in zip(xs, dys))


def _check(got, want, what):
    e = O.rel_err(got.cpu(), want.cpu())
    Cout, k = want.shape[0], want.shape[2]
    loc = max(O.rel_err(got[n0:n0 + 64, :, t // k, t % k].cpu(), want[n0:n0 + 64, :, t // k, t % k].cpu())
              for n0 in range(0, Cout, 64) for t in range(k * k))
    print('%s: rel err %.2e (bound %.0e), worst 64-channel x tap block %.2e (bound %.0e)' % (what, e, TOL_TC, loc, TOL_LOCAL))
    assert e < TOL_TC, (what, e)
    assert loc < TOL_LOCAL, (what, loc)


def _dw0(want, seed):
    g = torch.Generator(device=_dev()).manual_seed(seed)
    return torch.randn(want.shape, device=_dev(), generator=g) * float(want.std())


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['bf16x3', 'bf16'])
@pytest.mark.parametrize('Cin,Cout', BENCH_PAIRS)
def test_bench_plan_parity(ops, mode, Cin, Cout):
    """wgrad_planes_multi over P3..P7 at B = 32 (43 splits of at most 64 pixel boxes for the 256-channel inputs)"""
    ops.PRECISION = mode
    B = 32
    g = torch.Generator(device=_dev()).manual_seed(Cin * 1000 + Cout)
    xs = [torch.randn(B, h, w, Cin, device=_dev(), generator=g) for h, w in D0_512]
    dys = [torch.randn(B, h, w, Cout, device=_dev(), generator=g) for h, w in D0_512]
    xp, dyp = [_planes(ops, x) for x in xs], [_planes(ops, d) for d in dys]
    if mode == 'bf16':                     # the operands the single bf16 product sees
        xs = [p[0][..., :Cin].float() for p in xp]
        dys = [p[0][..., :Cout].float() for p in dyp]
    want = _ref(xs, dys, 3)
    del xs, dys
    dw0 = _dw0(want, 7)
    dw = dw0.clone()
    ops.wgrad_planes_multi(dw, [dict(x=xp[i], dy=dyp[i], B=B, H=h, W=w) for i, (h, w) in enumerate(D0_512)], dw, Cin, Cout, 3)
    _check(dw.double() - dw0.double(), want, 'wgrad %d->%d %s' % (Cin, Cout, mode))


def _fp32_levels(ops, maps, Cin, Cout, k, seed):
    """conv_wgrad_multi with a bias gradient on NHWC fp32 maps; -> (dw - dw0, dbias - db0, fp64 dw, fp64 dbias)"""
    ops.PRECISION = 'bf16x3'
    g = torch.Generator(device=_dev()).manual_seed(seed)
    xs = [torch.randn(B, h, w, Cin, device=_dev(), generator=g) for B, h, w in maps]
    dys = [torch.randn(B, h, w, Cout, device=_dev(), generator=g) for B, h, w in maps]
    want = _ref(xs, dys, k)
    want_b = sum(d.double().sum((0, 1, 2)) for d in dys)
    dw0, db0 = _dw0(want, seed + 1), _dw0(want_b, seed + 2)
    dw, db = dw0.clone(), db0.clone()
    lv = [dict(x_ptr=x.data_ptr(), x_bs=h * w * Cin, dy_ptr=d.data_ptr(), dy_bs=h * w * Cout, B=B, H=h, W=w)
          for x, d, (B, h, w) in zip(xs, dys, maps)]
    ops.conv_wgrad_multi(dw, lv, dw, db, Cin, Cout, k, tc=True)
    return dw.double() - dw0.double(), db.double() - db0.double(), want, want_b


@pytest.mark.gpu
@pytest.mark.parametrize('maps', [[(4, 16, 16)], [(2, 2, 2)]], ids=['tma', 'gather'])
def test_1x1_with_bias_reduces_into_dw(ops, maps):
    """a 1x1 weight gradient with a bias gradient takes a tensor-core kernel (the TMA-fed one when the map has a pixel
    box, the gathering one when not) that reduces into dw itself: no ws_dw is passed"""
    assert ops.pixel_boxes_ok(maps) == (maps[0][1] == 16)
    got, got_b, want, want_b = _fp32_levels(ops, maps, 64, 128, 1, 11)
    _check(got, want, '1x1 64->128 %s' % (maps,))
    assert O.rel_err(got_b.cpu(), want_b.cpu()) < 1e-5


@pytest.mark.gpu
def test_3x3_both_routes_one_fold(ops):
    """a 3x3 call whose 16x16 level takes the TMA-fed kernel and whose 2x2 level (no pixel box) takes the gathering one:
    both add into the one ws_dw, folded into dw once"""
    maps = [(2, 16, 16), (2, 2, 2)]
    assert ops.pixel_boxes_ok(maps[:1]) and not ops.pixel_boxes_ok(maps[1:])
    got, got_b, want, want_b = _fp32_levels(ops, maps, 96, 160, 3, 21)
    _check(got, want, '3x3 96->160 %s' % (maps,))
    assert O.rel_err(got_b.cpu(), want_b.cpu()) < 1e-5


def test_3x3_tensor_core_call_needs_ws_dw():
    """the refusal comes after every level's own checks and before any device work, so it runs without a GPU"""
    import __graft_entry__ as entry
    entry.build()
    from models import _native as N
    lib = N.load()
    fake = 1 << 20                                           # aligned non-null "pointer"; never dereferenced

    def wg(**kw):
        a = N.WgradArgs(x=fake, x_bstride=8 * 8 * 64, dy=fake, dy_bstride=8 * 8 * 64, dw=fake, B=2, H=8, W=8, Cin=64,
                        Cout=64, ksize=3, precision=1, ws_x=fake, ws_dy=fake)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def err():
        return lib.effdet_last_error().decode()

    assert lib.effdet_conv2d_wgrad(ctypes.byref(wg()), 0, None) == -1 and 'ws_dw' in err()
    assert lib.effdet_conv2d_wgrad(ctypes.byref(wg(ws_x=None, ws_dy=None)), 0, None) == -1 and 'ws_dw' in err()
    arr = (N.WgradArgs * 2)(wg(), wg(H=2, W=2))
    assert lib.effdet_conv2d_wgrad_multi(arr, 2, 0, None) == -1 and 'ws_dw' in err()
    arr = (N.WgradArgs * 2)(wg(), wg(B=0))                   # a level's own refusal comes first
    assert lib.effdet_conv2d_wgrad_multi(arr, 2, 0, None) == -1 and err() == 'wgrad: empty shape'
    assert lib.effdet_conv2d_wgrad(ctypes.byref(wg(ws_dw=fake + 4)), 0, None) == -1 and err() == \
        'wgrad: pointers must be 16-byte aligned'
