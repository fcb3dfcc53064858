"""Which kernel a dense convolution lands on, and that every route computes the same thing: inputs the tensor-core
kernels do not take reach the CUDA-core kernels, and one pyramid level through the multi-level entry points equals the
single-level call.  Needs an H100: every test is marked ``gpu``."""
import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O

pytestmark = pytest.mark.gpu

TOL_EXACT = 5e-5    # exact-fp32 CUDA-core kernels (summation order only)
TOL_TC = 3e-5       # bf16x3 split precision on the tensor cores


def _dev():
    return torch.device('cuda:0')


def _ops():
    from models import _ops as ops
    return ops


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(_dev())


def _nchw(y):
    return y.detach().permute(0, 3, 1, 2).contiguous().cpu()


def _swish(x):
    return x * torch.sigmoid(x)


def test_conv1x1_mbconv_inputs_on_strided_x_match_torch():
    """1x1 conv with the MBConv prologue (in_scale/in_shift, a_scale) and epilogue (z, scale/shift, row_scale) inputs
    and a tensor-core weight pack, on an x whose images lie 12 floats apart: the pointwise GEMM wants a dense x and the
    implicit-GEMM tensor-core kernel takes none of these inputs, so the CUDA-core kernel computes it."""
    ops = _ops()
    from models._native import ACT_SWISH
    N = ops.N
    dev = _dev()
    B, H, W, Cin, Cout = 3, 9, 7, 48, 40
    g = torch.Generator().manual_seed(17)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5
    isc, ish = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
    gate = torch.rand(B, Cin, generator=g)
    sc, sh = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g)
    rows = torch.tensor([0.0, 1.25, 0.8])
    res = torch.randn(B, Cout, H, W, generator=g)
    wp = torch.nn.Parameter(w.to(dev))
    wf, _ = ops.pack_conv(wp)
    tf = ops.pack_conv_tc(wp)[0]
    xs = H * W * Cin + 12
    xbuf = torch.full((B, xs), float('nan'), device=dev)
    xbuf[:, :H * W * Cin] = _nhwc(x).reshape(B, -1)
    y = torch.empty(B, H, W, Cout, device=dev)
    z = torch.empty(B, H, W, Cout, device=dev)
    resd = _nhwc(res)
    ys = H * W * Cout
    ops.conv2d_raw(xbuf, N.f32(xbuf), xs, wf, N.f32(y), ys, B, H, W, Cin, Cout, 1, z_ptr=N.f32(z), scale=sc.to(dev),
                   shift=sh.to(dev), a_scale=gate.to(dev), row_scale=rows.to(dev), res_ptr=N.f32(resd), res_bs=ys,
                   act=ACT_SWISH, w_tc=tf, in_scale=isc.to(dev), in_shift=ish.to(dev))
    a = _swish(x * isc[None, :, None, None] + ish[None, :, None, None]) * gate[:, :, None, None]
    z_ref = F.conv2d(a, w)
    y_ref = _swish(z_ref * sc[None, :, None, None] + sh[None, :, None, None]) * rows[:, None, None, None] + res
    assert O.rel_err(_nchw(z), z_ref) < TOL_EXACT
    assert O.rel_err(_nchw(y), y_ref) < TOL_EXACT


@pytest.mark.parametrize('B,H,W,Cin,Cout', [(2, 8, 8, 44, 24), (3, 5, 7, 20, 64)])
def test_conv1x1_wgrad_input_prologue_cin_not_multiple_of_8(B, H, W, Cin, Cout):
    """Weight gradient of a project conv (operand swish(bn(z)) * gate) with Cin % 8 == 4 and the tensor-core mode
    asked for: the pointwise weight-gradient kernel needs Cin % 8 == 0 and the TMA-fed one has no input prologue, so the
    CUDA-core kernel computes it."""
    ops = _ops()
    dev = _dev()
    g = torch.Generator().manual_seed(B + Cin + Cout)
    z = torch.randn(B, Cin, H, W, generator=g)
    dy = torch.randn(B, Cout, H, W, generator=g)
    isc, ish = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
    gate = torch.rand(B, Cin, generator=g)
    a = _swish(z * isc[None, :, None, None] + ish[None, :, None, None]) * gate[:, :, None, None]
    wr = torch.zeros(Cout, Cin, 1, 1, requires_grad=True)
    F.conv2d(a, wr).backward(dy)
    dw = torch.zeros(Cout, Cin, 1, 1, device=dev)
    ops.conv_wgrad(_nhwc(z), _nhwc(dy), dw, None, 1, a_scale=gate.to(dev), tc=True, in_scale=isc.to(dev),
                   in_shift=ish.to(dev))
    assert O.rel_err(dw.cpu(), wr.grad) < TOL_EXACT


def test_conv3x3_single_and_multi_level_are_bit_identical():
    """conv2d on each map and conv2d_multi over one and over several maps run the same tensor-core kernel: the
    outputs are bit-identical.  The 2x2 map has no TMA pixel box, the case the fp32-input kernel exists for."""
    ops = _ops()
    from models._native import ACT_RELU
    lib = ops.N.load()
    dev = _dev()
    Cin, Cout = 64, 88
    shapes = [(2, 2, 2), (2, 5, 3), (2, 8, 8)]
    assert not lib.effdet_wgrad_tc_geometry_ok(*shapes[0])
    g = torch.Generator().manual_seed(23)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (Cin * 9) ** 0.5
    b = torch.randn(Cout, generator=g)
    xs = [torch.randn(B, Cin, H, W, generator=g) for B, H, W in shapes]
    wp = torch.nn.Parameter(w.to(dev))
    wf, _ = ops.pack_conv(wp)
    tf = ops.pack_conv_tc(wp)[0]
    bd = b.to(dev)
    xd = [_nhwc(x) for x in xs]
    single = [ops.conv2d(x, wf, Cout, 3, bias=bd, act=ACT_RELU, w_tc=tf) for x in xd]
    for x, y in zip(xd, single):
        assert torch.equal(ops.conv2d_multi([x], wf, Cout, 3, bias=bd, act=ACT_RELU, w_tc=tf)[0], y)
    multi = ops.conv2d_multi(xd, wf, Cout, 3, bias=bd, act=ACT_RELU, w_tc=tf)
    for x, y, ym in zip(xs, single, multi):
        assert torch.equal(ym, y)
        assert O.rel_err(_nchw(y), torch.relu(F.conv2d(x, w, b, 1, 1))) < TOL_TC


@pytest.mark.parametrize('Cin,Cout', [(64, 64), (256, 36)])
def test_wgrad_single_and_multi_level_agree(Cin, Cout):
    """The TMA-fed weight gradient over several pyramid levels in one launch equals the sum of one call per level
    (and torch), bias gradient included; the sums differ only in the order of the atomics."""
    ops = _ops()
    N = ops.N
    dev = _dev()
    shapes = [(2, 16, 16), (2, 8, 8), (2, 4, 4)]
    lib = N.load()
    assert all(lib.effdet_wgrad_tc_geometry_ok(*s) for s in shapes)
    g = torch.Generator().manual_seed(Cin + Cout)
    xs = [torch.randn(B, Cin, H, W, generator=g) for B, H, W in shapes]
    dys = [torch.randn(B, Cout, H, W, generator=g) for B, H, W in shapes]
    wr = torch.zeros(Cout, Cin, 3, 3, requires_grad=True)
    br = torch.zeros(Cout, requires_grad=True)
    sum(F.conv2d(x, wr, br, 1, 1).mul(dy).sum() for x, dy in zip(xs, dys)).backward()
    xd, dyd = [_nhwc(x) for x in xs], [_nhwc(dy) for dy in dys]
    dw1, db1 = torch.zeros(Cout, Cin, 3, 3, device=dev), torch.zeros(Cout, device=dev)
    for x, dy in zip(xd, dyd):
        ops.conv_wgrad(x, dy, dw1, db1, 3, tc=True)
    dwm, dbm = torch.zeros_like(dw1), torch.zeros_like(db1)
    levels = [dict(x_ptr=N.f32(x), x_bs=H * W * Cin, dy_ptr=N.f32(dy), dy_bs=H * W * Cout, B=B, H=H, W=W)
              for x, dy, (B, H, W) in zip(xd, dyd, shapes)]
    ops.conv_wgrad_multi(xd[0], levels, dwm, dbm, Cin, Cout, 3, tc=True)
    assert O.rel_err(dwm.cpu(), dw1.cpu()) < TOL_TC
    assert O.rel_err(dbm.cpu(), db1.cpu()) < TOL_EXACT
    assert O.rel_err(dwm.cpu(), wr.grad) < TOL_TC and O.rel_err(dw1.cpu(), wr.grad) < TOL_TC
    assert O.rel_err(dbm.cpu(), br.grad) < TOL_EXACT
