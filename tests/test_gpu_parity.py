"""Parity of the CUDA hot path (through the C ABI / nn.Module mirror) against the CPU oracle and the
golden vectors captured from the real reference.  Needs an H100: every test is marked ``gpu``.

Metric: per-tensor norm-relative error ||a-b||_2/||b||_2 (SURVEY.md 8(c)).  north_star's bar is
1e-3 (fp32); the exact-fp32 CUDA-core kernels are held to TOL_EXACT, integer outputs (anchors,
NMS keep sets, class ids) to bit equality.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-3          # north_star tolerance (forward outputs, losses)
TOL_EXACT = 5e-5    # what the exact-fp32 kernels must reach (atomics / summation order only)
# End-to-end GRADIENT tolerance.  Gradients of this network are ill-conditioned w.r.t. forward round-off:
# tools/grad_conditioning.py multiplies every conv output of
# the fp32 CPU oracle by (1 + 5e-6 * N(0,1)) -- the per-layer error the bf16x3 tensor-core products measure at
# (test_conv2d_tensor_core_forward_dgrad_wgrad holds them to 3e-5) -- and the worst parameter gradient moves by 1.3e-2
# (amplification ~2600x: the regression tower, where smooth-L1 / ReLU decisions sit within round-off of their
# switching point), the median one by 2.8e-4.  The bf16x3 bound below is that noise level times 1.5; the exact-fp32
# path carries ~1e-7 per layer.
TOL_GRAD = {'fp32': 5e-3, 'bf16x3': 2e-2}
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _dev():
    return torch.device('cuda:0')


@pytest.fixture(params=['bf16x3', 'fp32'])
def prec(request):
    """run a test under both conv precisions of the product (tensor cores / exact fp32 CUDA cores)"""
    from models import _ops as ops
    old = ops.PRECISION
    ops.PRECISION = request.param
    yield request.param
    ops.PRECISION = old


def _ops():
    from models import _ops as ops
    return ops


def _rel(a, b):
    return O.rel_err(a, b)


def _nhwc(x):   # NCHW cpu -> NHWC cuda contiguous
    return x.permute(0, 2, 3, 1).contiguous().to(_dev())


def _nchw(y):   # NHWC cuda -> NCHW cpu
    return y.detach().permute(0, 3, 1, 2).contiguous().cpu()


# ------------------------------------------------------------------------------------------------
# single kernels
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('B,H,W,Cin,Cout,k', [
    (2, 16, 16, 64, 64, 3), (1, 8, 8, 256, 256, 3), (2, 4, 4, 256, 720, 3), (3, 8, 8, 256, 36, 3),
    (2, 32, 32, 16, 96, 1), (2, 16, 16, 144, 24, 1), (1, 16, 16, 40, 64, 1), (2, 7, 5, 24, 40, 3),
    (5, 4, 4, 64, 256, 3), (2, 4, 4, 180, 256, 3), (2, 2, 2, 36, 256, 3),
])
def test_conv2d_forward_dgrad_wgrad(B, H, W, Cin, Cout, k):
    ops = _ops()
    g = torch.Generator().manual_seed(B * 1000 + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g)
    dy = torch.randn(B, Cout, H, W, generator=g)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = F.conv2d(xr, wr, br, 1, k // 2)
    yr.backward(dy)
    wp = torch.nn.Parameter(w.to(_dev()))
    wf, wd = ops.pack_conv(wp)
    xd, dyd = _nhwc(x), _nhwc(dy)
    y = ops.conv2d(xd, wf, Cout, k, bias=b.to(_dev()))
    assert _rel(_nchw(y), yr) < TOL_EXACT
    dx = ops.conv2d(dyd, wd, Cin, k)
    assert _rel(_nchw(dx), xr.grad) < TOL_EXACT
    dw = torch.zeros(Cout, Cin, k, k, device=_dev())
    db = torch.zeros(Cout, device=_dev())
    ops.conv_wgrad(xd, dyd, dw, db, k)
    assert _rel(dw.cpu(), wr.grad) < TOL_EXACT
    assert _rel(db.cpu(), br.grad) < TOL_EXACT


TOL_TC = 3e-5       # bf16x3 split precision on the tensor cores (~2^-16 per product, fp32 accumulate)


@pytest.mark.parametrize('B,H,W,Cin,Cout,k', [
    (2, 16, 16, 64, 64, 3), (1, 8, 8, 256, 256, 3), (2, 4, 4, 256, 720, 3), (3, 8, 8, 256, 36, 3),
    (2, 16, 16, 64, 256, 3), (2, 8, 8, 720, 256, 3), (2, 8, 8, 36, 256, 3), (1, 16, 16, 40, 64, 1),
    (5, 4, 4, 256, 64, 3), (2, 7, 5, 88, 88, 3), (4, 32, 32, 256, 256, 3), (2, 32, 32, 16, 96, 1),
    (2, 16, 16, 144, 24, 1), (2, 8, 8, 192, 1152, 1), (2, 8, 8, 480, 112, 1),
])
def test_conv2d_tensor_core_forward_dgrad_wgrad(B, H, W, Cin, Cout, k):
    """wgmma bf16x3 implicit GEMM (fwd, dgrad through the rotated pack, wgrad) vs torch fp32 conv."""
    ops = _ops()
    from models._native import ACT_RELU
    g = torch.Generator().manual_seed(B * 1000 + Cin + Cout + 7)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=g)
    dy = torch.randn(B, Cout, H, W, generator=g)
    res = torch.randn(B, Cout, H, W, generator=g)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    yr = F.conv2d(xr, wr, br, 1, k // 2)
    yr.backward(dy)
    wp = torch.nn.Parameter(w.to(_dev()))
    wf, wd = ops.pack_conv(wp)
    tf, td = ops.pack_conv_tc(wp)
    xd, dyd = _nhwc(x), _nhwc(dy)
    y = ops.conv2d(xd, wf, Cout, k, bias=b.to(_dev()), w_tc=tf)
    e_f = _rel(_nchw(y), yr)
    y2 = ops.conv2d(xd, wf, Cout, k, bias=b.to(_dev()), act=ACT_RELU, residual=_nhwc(res), mask_src=_nhwc(dy), w_tc=tf)
    e_e = _rel(_nchw(y2), (torch.relu(yr.detach()) + res) * (dy > 0))
    dx = ops.conv2d(dyd, wd, Cin, k, w_tc=td)
    e_d = _rel(_nchw(dx), xr.grad)
    dw = torch.zeros(Cout, Cin, k, k, device=_dev())
    db = torch.zeros(Cout, device=_dev())
    ops.conv_wgrad(xd, dyd, dw, db, k, tc=True)
    e_w = _rel(dw.cpu(), wr.grad)
    print('tc conv %s fwd %.2e epi %.2e dgrad %.2e wgrad %.2e' % ((B, H, W, Cin, Cout, k), e_f, e_e, e_d, e_w))
    assert e_f < TOL_TC and e_e < TOL_TC and e_d < TOL_TC
    assert e_w < TOL_TC
    assert _rel(db.cpu(), br.grad) < TOL_EXACT


@pytest.mark.parametrize('use_tc', [False, True])
def test_conv2d_epilogue_options(use_tc):
    ops = _ops()
    from models._native import ACT_RELU, ACT_SIGMOID, ACT_SWISH
    g = torch.Generator().manual_seed(5)
    B, H, W, Cin, Cout = 3, 8, 8, 48, 40
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5
    scale, shift = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g)
    gate = torch.rand(B, Cin, generator=g)
    rows = torch.tensor([0.0, 1.25, 1.25])
    res = torch.randn(B, Cout, H, W, generator=g)
    wpar = torch.nn.Parameter(w.to(_dev()))
    wf, _ = ops.pack_conv(wpar)
    tcw = ops.pack_conv_tc(wpar)[0] if use_tc else None
    tol = TOL_TC if use_tc else TOL_EXACT
    xd = _nhwc(x)
    z_ref = F.conv2d(x * gate[:, :, None, None], w)
    u = z_ref * scale[None, :, None, None] + shift[None, :, None, None]
    y, z = ops.conv2d(xd, wf, Cout, 1, scale=scale.to(_dev()), shift=shift.to(_dev()), a_scale=gate.to(_dev()),
                      row_scale=rows.to(_dev()), residual=_nhwc(res), act=ACT_SWISH, save_z=True, w_tc=tcw)
    assert _rel(_nchw(z), z_ref) < tol
    assert _rel(_nchw(y), O.swish(u) * rows[:, None, None, None] + res) < tol
    y = ops.conv2d(xd, wf, Cout, 1, act=ACT_SIGMOID, w_tc=tcw)
    assert _rel(_nchw(y), torch.sigmoid(F.conv2d(x, w))) < tol
    y = ops.conv2d(xd, wf, Cout, 1, act=ACT_RELU, mask_src=_nhwc(res), w_tc=tcw)
    assert _rel(_nchw(y), torch.relu(F.conv2d(x, w)) * (res > 0)) < tol


def _swish(x):
    return x * torch.sigmoid(x)


@pytest.mark.parametrize('k,s,pre,C,H,W,B', [
    (3, 1, True, 24, 20, 36, 2), (5, 1, True, 40, 16, 16, 2), (3, 2, True, 96, 32, 32, 2), (5, 2, True, 144, 24, 40, 1),
    (3, 1, False, 32, 33, 17, 2), (5, 2, True, 20, 9, 7, 3), (3, 2, True, 16, 7, 11, 2), (5, 1, True, 1152, 8, 8, 2),
    (3, 2, True, 1152, 8, 8, 2), (5, 1, False, 16, 40, 20, 1),
])
def test_dwconv_fused_forward_backward(k, s, pre, C, H, W, B):
    """effdet_dwconv_fwd_fused / effdet_dwconv_bwd_fused (pre-activation-only MBConv depthwise phase) against torch
    autograd on the CPU: z1, the squeeze-excite mean, and from (dq, gate, dmean) the gradients of the raw input,
    the depthwise weight and both BatchNorm affines -- odd sizes, tile tails, stride-2 polyphase, 1152 channels."""
    from models import _native as N
    ops = _ops()
    dev = _dev()
    g = torch.Generator().manual_seed(k * 100 + s * 10 + C + H)
    eps = 1e-3
    pt = (k - 1) // 2 if s == 1 else (0 if k == 3 else 1)
    total = {(3, 1): 2, (3, 2): 1, (5, 1): 4, (5, 2): 3}[(k, s)]
    Ho, Wo = (H + total - k) // s + 1, (W + total - k) // s + 1
    x = torch.randn(B, C, H, W, generator=g)
    wd = torch.randn(C, 1, k, k, generator=g) / k
    bn = [dict(g=torch.rand(C, generator=g) + 0.5, b=torch.randn(C, generator=g) * 0.3, m=torch.randn(C, generator=g) * 0.3,
               v=torch.rand(C, generator=g) + 0.5) for _ in range(2)]
    gate = torch.rand(B, C, generator=g)
    dq = torch.randn(B, C, Ho, Wo, generator=g)
    dmean = torch.randn(B, C, generator=g)
    # ---- torch reference ----
    xr = x.clone().requires_grad_(True)
    wr = wd.clone().requires_grad_(True)
    gam = [b_['g'].clone().requires_grad_(True) for b_ in bn]
    bet = [b_['b'].clone().requires_grad_(True) for b_ in bn]

    def bnf(t, i):
        return F.batch_norm(t, bn[i]['m'], bn[i]['v'], gam[i], bet[i], False, 0.0, eps)
    a0 = _swish(bnf(xr, 0)) if pre else xr
    z1r = F.conv2d(F.pad(a0, (pt, total - pt, pt, total - pt)), wr, None, s, 0, 1, C)
    a1 = _swish(bnf(z1r, 1))
    meanr = a1.mean(dim=(2, 3))
    ((a1 * gate[:, :, None, None] * dq).sum() + (meanr * dmean).sum()).backward()
    # ---- kernels ----
    def fold(i):
        rstd = 1.0 / torch.sqrt(bn[i]['v'] + eps)
        sc = bn[i]['g'] * rstd
        return [t.to(dev).contiguous() for t in (sc, bn[i]['b'] - bn[i]['m'] * sc, bn[i]['m'], rstd)]
    sc0, sh0, mu0, rs0 = fold(0)
    sc1, sh1, mu1, rs1 = fold(1)
    xd = _nhwc(x)
    wkkc = wd.view(C, k * k).t().contiguous().to(dev)
    z1 = torch.empty(B, Ho, Wo, C, device=dev)
    mean = torch.zeros(B, C, device=dev)
    fa = N.DwFwdArgs(N.f32(xd), N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(wkkc), N.f32(sc1), N.f32(sh1),
                     N.f32(z1), N.f32(mean), B, H, W, C, k, s, pt, pt, Ho, Wo, 1.0 / (Ho * Wo))
    N.call('effdet_dwconv_fwd_fused', xd, fa)
    assert _rel(_nchw(z1), z1r.detach()) < TOL_EXACT
    assert _rel(mean.cpu(), meanr.detach()) < TOL_EXACT
    dqd, gated, dmd = _nhwc(dq), gate.to(dev), dmean.to(dev)
    dx = torch.full((B, H, W, C), float('nan'), device=dev)
    dw = torch.zeros(C, 1, k, k, device=dev)
    dgb = torch.zeros(4, C, device=dev)
    ba = N.DwBwdArgs(N.f32(dqd), N.f32(z1), N.f32(gated), N.f32(dmd), N.f32(sc1), N.f32(sh1), N.f32(mu1), N.f32(rs1), N.f32(xd),
                     N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(mu0) if pre else None,
                     N.f32(rs0) if pre else None, N.f32(wkkc), N.f32(dx), N.f32(dw), N.f32(dgb[0]), N.f32(dgb[1]),
                     N.f32(dgb[2]) if pre else None, N.f32(dgb[3]) if pre else None, 1.0 / (Ho * Wo), B, H, W, C, k, s, pt, pt,
                     Ho, Wo, None)
    N.call('effdet_dwconv_bwd_fused', xd, ba)
    errs = dict(dx=_rel(_nchw(dx), xr.grad), dw=_rel(dw.cpu(), wr.grad), dg1=_rel(dgb[0].cpu(), gam[1].grad),
                db1=_rel(dgb[1].cpu(), bet[1].grad))
    if pre:
        errs.update(dg0=_rel(dgb[2].cpu(), gam[0].grad), db0=_rel(dgb[3].cpu(), bet[0].grad))
    assert max(errs.values()) < TOL_EXACT, errs
    if pre and C % 8 == 0:                                   # same kernel writing dx as bf16 hi/lo planes instead of fp32
        planes = torch.full((2, B, H, W, C), float('nan'), device=dev, dtype=torch.bfloat16)
        dw2, dgb2 = torch.zeros_like(dw), torch.zeros_like(dgb)
        ba.dx, ba.dx_planes, ba.dw = None, planes.data_ptr(), N.f32(dw2)
        ba.dgamma1, ba.dbeta1, ba.dgamma0, ba.dbeta0 = (N.f32(dgb2[i]) for i in range(4))
        N.call('effdet_dwconv_bwd_fused', xd, ba)
        assert _rel((planes[0].float() + planes[1].float()).permute(0, 3, 1, 2).cpu(), xr.grad) < 3e-5
        assert _rel(dw2.cpu(), wr.grad) < TOL_EXACT
    # gradient w.r.t. the SE gate with the activation recomputed from the raw tensor
    dgate = torch.zeros(B, C, device=dev)
    N.call('effdet_spatial_reduce_act', xd, N.f32(dqd), N.f32(z1), N.f32(sc1), N.f32(sh1), N.f32(dgate), 1.0, B, Ho * Wo, C)
    want = (dq * a1.detach()).sum(dim=(2, 3))
    assert _rel(dgate.cpu(), want) < TOL_EXACT


@pytest.mark.parametrize('B,H,W,Cin,Cout', [(2, 16, 16, 96, 24), (1, 12, 20, 144, 40), (2, 8, 8, 1152, 192), (3, 9, 7, 32, 16)])
def test_conv1x1_input_prologue(B, H, W, Cin, Cout, prec):
    """project conv of the pre-activation-only MBConv: operand = swish(bn(z)) * gate built while the tile is staged
    (effdet_conv_args.in_scale/in_shift/a_scale), forward and weight gradient, both precisions"""
    ops = _ops()
    dev = _dev()
    g = torch.Generator().manual_seed(B + Cin + Cout)
    z = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5
    sc, sh = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
    gate = torch.rand(B, Cin, generator=g)
    dy = torch.randn(B, Cout, H, W, generator=g)
    a = _swish(z * sc[None, :, None, None] + sh[None, :, None, None]) * gate[:, :, None, None]
    wr = w.clone().requires_grad_(True)
    yr = F.conv2d(a, wr)
    yr.backward(dy)
    wp = torch.nn.Parameter(w.to(dev))
    wf, _ = ops.pack_conv(wp)
    tf = ops.tc_packs(wp)[0]
    zd = _nhwc(z)
    y = ops.conv2d(zd, wf, Cout, 1, a_scale=gate.to(dev), in_scale=sc.to(dev), in_shift=sh.to(dev), w_tc=tf)
    tol = TOL_EXACT if prec == 'fp32' else TOL_TC
    assert _rel(_nchw(y), yr.detach()) < tol
    dw = torch.zeros(Cout, Cin, 1, 1, device=dev)
    ops.conv_wgrad(zd, _nhwc(dy), dw, None, 1, a_scale=gate.to(dev), tc=ops.tc_enabled(), in_scale=sc.to(dev),
                   in_shift=sh.to(dev))
    assert _rel(dw.cpu(), wr.grad) < tol


@pytest.mark.parametrize('B,H,W,Cin,Cout', [
    (2, 64, 64, 16, 96), (1, 100, 37, 24, 144), (2, 16, 16, 144, 24), (2, 8, 8, 1152, 192), (2, 8, 8, 192, 1152),
    (3, 20, 12, 40, 240), (2, 16, 16, 672, 112), (1, 8, 8, 320, 64), (8, 64, 64, 32, 16), (5, 48, 48, 96, 24),
    (1, 3, 5, 80, 480), (2, 32, 32, 480, 80),
])
def test_pointwise_gemm_persistent_kernel(B, H, W, Cin, Cout):
    """pw_gemm_kernel (persistent TMA-fed wgmma GEMM of every backbone / lateral 1x1 conv) vs torch fp32: the three
    epilogue routes -- plain output through TMA tile stores, bias, and the MBConv project epilogue (raw-output save,
    BN affine, drop-connect scale, residual) with direct stores -- over row tails, several n-tiles, 1..18 k-blocks
    and more m-tiles than CTAs."""
    ops = _ops()
    dev = _dev()
    g = torch.Generator().manual_seed(B * 1000 + Cin + Cout + 11)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5
    bias = torch.randn(Cout, generator=g)
    sc, sh = torch.rand(Cout, generator=g) + 0.5, torch.randn(Cout, generator=g)
    rsc = torch.rand(B, generator=g) + 0.5
    res = torch.randn(B, Cout, H, W, generator=g)
    wp = torch.nn.Parameter(w.to(dev))
    wf, wd = ops.pack_conv(wp)
    tf, td = ops.pack_conv_tc(wp)
    xd = _nhwc(x)
    ref = F.conv2d(x, w)
    y = ops.conv2d(xd, wf, Cout, 1, w_tc=tf)                                   # plain: TMA-store epilogue
    assert _rel(_nchw(y), ref) < TOL_TC
    y = ops.conv2d(xd, wf, Cout, 1, bias=bias.to(dev), w_tc=tf)                # lateral conv: + bias
    assert _rel(_nchw(y), ref + bias[None, :, None, None]) < TOL_TC
    y, z = ops.conv2d(xd, wf, Cout, 1, scale=sc.to(dev), shift=sh.to(dev), row_scale=rsc.to(dev), residual=_nhwc(res),
                      save_z=True, w_tc=tf)                                    # project conv epilogue, direct stores
    want = (ref * sc[None, :, None, None] + sh[None, :, None, None]) * rsc[:, None, None, None] + res
    assert _rel(_nchw(z), ref) < TOL_TC and _rel(_nchw(y), want) < TOL_TC
    dy = torch.randn(B, Cout, H, W, generator=g)                               # data gradient = same kernel, transposed pack
    dx = ops.conv2d(_nhwc(dy), wd, Cin, 1, w_tc=td)
    assert _rel(_nchw(dx), F.conv_transpose2d(dy, w)) < TOL_TC


@pytest.mark.parametrize('B,H,W,Cin,Cexp', [(2, 32, 32, 16, 96), (1, 64, 64, 24, 144), (2, 16, 16, 80, 480), (3, 8, 8, 192, 1152)])
def test_expand_gradients_from_bf16_planes(B, H, W, Cin, Cexp):
    """The gradient of the expand conv's raw output exists only as bf16 hi/lo planes (written by
    effdet_dwconv_bwd_fused): data gradient (pw_gemm_kernel, planes mode: TMA straight into the MMA operand layout)
    and weight gradient (TMA-fed kernel, no split pass) from planes vs torch fp32."""
    ops = _ops()
    dev = _dev()
    assert ops.planes_ok(B, H, W, Cexp)
    g = torch.Generator().manual_seed(B + Cin + Cexp)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cexp, Cin, 1, 1, generator=g) / Cin ** 0.5
    dz = torch.randn(B, Cexp, H, W, generator=g)
    res = torch.randn(B, Cin, H, W, generator=g)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    F.conv2d(xr, wr).backward(dz)
    dzd = _nhwc(dz)
    hi = dzd.to(torch.bfloat16)
    lo = (dzd - hi.float()).to(torch.bfloat16)
    planes = torch.stack([hi, lo]).contiguous()
    wp = torch.nn.Parameter(w.to(dev))
    _, wd = ops.pack_conv(wp)
    td = ops.tc_packs(wp)[1]
    dx = ops.conv2d_from_planes(planes, wd, Cin, residual=_nhwc(res), w_tc=td)
    assert _rel(_nchw(dx), xr.grad + res) < TOL_TC
    dw = torch.zeros(Cexp, Cin, 1, 1, device=dev)
    xd = _nhwc(x)
    ops.conv_wgrad_raw(xd, ops.N.f32(xd), H * W * Cin, None, H * W * Cexp, dw, None, B, H, W, Cin, Cexp, 1, tc=True, dy_planes=planes)
    assert _rel(dw.cpu(), wr.grad) < TOL_TC


@pytest.mark.parametrize('B,H,W,Cin,Cout,mode', [
    (2, 16, 16, 144, 24, 'project'), (1, 4, 4, 32, 16, 'project'), (3, 10, 10, 96, 24, 'project'),
    (2, 8, 8, 1152, 192, 'project'), (2, 8, 8, 1152, 320, 'project'), (5, 9, 7, 240, 40, 'plain'),
    (2, 32, 32, 16, 96, 'planes'), (3, 8, 8, 192, 1152, 'planes'), (1, 16, 16, 112, 672, 'plain'),
    (2, 16, 16, 24, 144, 'plain'), (40, 32, 32, 40, 240, 'planes'), (1, 5, 3, 8, 8, 'plain'),
])
def test_pointwise_wgrad_fused_kernel(B, H, W, Cin, Cout, mode):
    """pw_wgrad_kernel: weight gradient of a 1x1 conv straight from the fp32 tensors (converter warps apply the
    BN+swish+SE-gate prologue and split to bf16 hi/lo in shared memory; GEMM-K = pixels) vs torch fp32 -- pixel tails
    that are not a multiple of the 64-pixel stage, several input-channel tiles (Cin > 256), several output-channel
    tiles (Cout > 128), dy given as fp32 or as bf16 planes, accumulation into a non-zero dw."""
    ops = _ops()
    dev = _dev()
    g = torch.Generator().manual_seed(B * 77 + Cin + Cout)
    x = torch.randn(B, Cin, H, W, generator=g)
    dy = torch.randn(B, Cout, H, W, generator=g)
    w = torch.randn(Cout, Cin, 1, 1, generator=g) / Cin ** 0.5
    sc, sh = torch.rand(Cin, generator=g) + 0.5, torch.randn(Cin, generator=g) * 0.3
    gate = torch.rand(B, Cin, generator=g)
    a = x
    if mode == 'project':
        a = _swish(x * sc[None, :, None, None] + sh[None, :, None, None]) * gate[:, :, None, None]
    wr = w.clone().requires_grad_(True)
    F.conv2d(a, wr).backward(dy)
    dw0 = torch.randn(Cout, Cin, 1, 1, generator=g)
    dw = dw0.clone().to(dev)
    xd, dyd = _nhwc(x), _nhwc(dy)
    kw = {}
    if mode == 'project':
        kw = dict(a_scale=gate.to(dev), in_scale=sc.to(dev), in_shift=sh.to(dev))
    if mode == 'planes':
        hi = dyd.to(torch.bfloat16)
        lo = (dyd - hi.float()).to(torch.bfloat16)
        planes = torch.stack([hi, lo]).contiguous()
        if not ops.planes_ok(B, H, W, Cout):
            pytest.skip('no pixel-box geometry for the fallback contract')
        ops.conv_wgrad_raw(xd, ops.N.f32(xd), H * W * Cin, None, H * W * Cout, dw, None, B, H, W, Cin, Cout, 1, tc=True,
                           dy_planes=planes)
    else:
        ops.conv_wgrad(xd, dyd, dw, None, 1, tc=True, **kw)
    assert _rel(dw.cpu() - dw0, wr.grad) < TOL_TC


def test_layout_transposes():
    from models import _ops as ops
    x = torch.randn(3, 24, 7, 9)
    xd = x.to(_dev()).requires_grad_(True)
    y = ops.to_nhwc(xd)
    assert torch.equal(y.detach().cpu(), x.permute(0, 2, 3, 1).contiguous())
    y.backward(torch.ones_like(y) * 2)
    assert torch.equal(xd.grad.cpu(), torch.full_like(x, 2.0))
    cl = x.to(_dev()).contiguous(memory_format=torch.channels_last)
    assert ops.to_nhwc(cl).data_ptr() == cl.data_ptr()          # zero-copy for channels_last input


# ------------------------------------------------------------------------------------------------
# modules vs oracle
# ------------------------------------------------------------------------------------------------

def _load(module, sd, prefix):
    sub = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    module.load_state_dict(sub)
    return module.to(_dev())


def _grad_sd(sd):
    return {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v)
            for k, v in sd.items()}


def _compare_param_grads(module, sdg, prefix, tol=TOL_EXACT, skip=()):
    worst = (0.0, None)
    for name, p in module.named_parameters():
        ref = sdg[prefix + name].grad
        if name in skip:
            continue
        if ref is None or float(ref.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) < 1e-12, name
            continue
        assert p.grad is not None, 'no gradient for ' + name
        e = _rel(p.grad, ref)
        if e > worst[0]:
            worst = (e, name)
        assert e < tol, (name, e)
    return worst


@pytest.mark.parametrize('net,size', [('efficientdet-d0', 128), ('efficientdet-d1', 128)])
def test_backbone_forward_backward(net, size, prec):
    from models.efficientnet import EfficientNet
    from models.efficientdet import MODEL_MAP
    cfg = O.make_config(net, 20, 64, 2)
    sd = O.init_state_dict(cfg, seed=11)
    m = _load(EfficientNet.from_name(MODEL_MAP[net], override_params={'num_classes': 1000}), sd, 'backbone.')
    m.eval()
    x, _ = O.synthetic_batch(2, size=size, seed=3)
    sdg = _grad_sd(sd)
    ref = O.backbone_forward(sdg, x, cfg)
    outs = m(x.to(_dev()))
    assert len(outs) == 7
    g = torch.Generator().manual_seed(1)
    loss_ref, loss = 0, 0
    for r, o in zip(ref, outs):
        assert tuple(o.shape) == tuple(r.shape)
        assert _rel(o.detach().cpu(), r.detach()) < (TOL_EXACT if prec == 'fp32' else 2e-4)
        wgt = torch.randn(r.shape, generator=g)
        loss_ref = loss_ref + (r * wgt).sum()
        loss = loss + (o * wgt.to(_dev())).sum()
    loss_ref.backward()
    loss.backward()
    worst = _compare_param_grads(m, sdg, 'backbone.', tol=2e-4 if prec == 'fp32' else 5e-3)
    print('backbone', prec, 'worst grad rel err', worst)


def test_drop_connect_uses_same_rng_stream():
    """train mode: the per-sample keep mask must consume torch.rand([B,1,1,1]) on the device in block
    order like the reference (models/utils.py:79-90); replay the same CUDA RNG stream for the oracle."""
    from models.efficientnet import EfficientNet
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    sd = O.init_state_dict(cfg, seed=12)
    m = _load(EfficientNet.from_name('efficientnet-b0'), sd, 'backbone.')
    m.train()
    for mod in m.modules():                            # train.py:100-102: train() then freeze_bn()
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eval()
    x, _ = O.synthetic_batch(4, size=128, seed=4)
    torch.manual_seed(1234)
    outs = m(x.to(_dev()))
    torch.manual_seed(1234)
    nskip = sum(1 for i, b in enumerate(cfg['blocks']) if b['skip'] and i > 0)
    keeps = [torch.rand([4, 1, 1, 1], dtype=torch.float32, device=_dev()).cpu() for _ in range(nskip)]
    with torch.no_grad():
        ref = O.backbone_forward(sd, x, cfg, keep_samples=keeps)
    for r, o in zip(ref, outs):
        assert _rel(o.detach().cpu(), r) < TOL_EXACT


@pytest.mark.parametrize('W,D,B', [(64, 2, 2), (88, 1, 2), (64, 2, 4), (224, 1, 4), (384, 1, 4)])
def test_bifpn_forward_backward(W, D, B, prec):
    """B=2: the 2x2 level has no legal TMA pixel box -> gather kernels; B=4: every level qualifies -> in tensor-core
    mode the fused maps are bf16 planes and the node convs run on conv_planes_kernel<64/128/256> (1 or 2 channel tiles)"""
    from models.bifpn import BIFPN
    cfg = O.make_config('efficientdet-d0', 20, W, D)
    sd = O.init_state_dict(cfg, seed=21)
    chans = cfg['stage_out'][-5:]
    m = _load(BIFPN(in_channels=chans, out_channels=W, stack=D, num_outs=5), sd, 'neck.')
    g = torch.Generator().manual_seed(2)
    feats = [torch.randn(B, c, 32 >> i, 32 >> i, generator=g) for i, c in enumerate(chans)]
    fr = [f.clone().requires_grad_(True) for f in feats]
    fd = [f.to(_dev()).requires_grad_(True) for f in feats]
    sdg = _grad_sd(sd)
    ref = O.bifpn_forward(sdg, fr, cfg)
    outs = m(fd)
    assert isinstance(outs, tuple) and len(outs) == 5
    lr, l = 0, 0
    ftol = TOL_EXACT if prec == 'fp32' else 2e-4
    gtol = 2e-4 if prec == 'fp32' else 5e-3
    for r, o in zip(ref, outs):
        assert _rel(o.detach().cpu(), r.detach()) < ftol
        wgt = torch.randn(r.shape, generator=g)
        lr = lr + (r * wgt).sum()
        l = l + (o * wgt.to(_dev())).sum()
    lr.backward()
    l.backward()
    for a, b in zip(fd, fr):
        assert _rel(a.grad.cpu(), b.grad) < gtol
    worst = _compare_param_grads(m, sdg, 'neck.', tol=gtol)
    print('bifpn', prec, 'worst grad rel err', worst)
    # fusion-weight gradients individually (tiny tensors, signed weights exercise the ReLU)
    for d in range(D):
        for wn in ('w1', 'w2'):
            k = 'stack_bifpn_convs.%d.%s' % (d, wn)
            assert _rel(dict(m.named_parameters())[k].grad, sdg['neck.' + k].grad) < gtol, k


def test_head_forward_backward(prec):
    from models.retinahead import RetinaHead
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    sd = O.init_state_dict(cfg, seed=31)
    m = _load(RetinaHead(num_classes=20, in_channels=64), sd, 'bbox_head.')
    # NB: a ReLU pre-activation within round-off of 0 can legitimately flip its mask between the CPU and
    # the CUDA summation order, which changes one gradient path outright (seen with seed 3 on the 4x4
    # level: 2e-3 on that level, 1e-6 everywhere else).  Seed 4 has no such coincidence.
    g = torch.Generator().manual_seed(4)
    feats = [torch.randn(2, 64, 16 >> i, 16 >> i, generator=g) for i in range(5)]
    feats[4] = torch.randn(2, 64, 1, 1, generator=g)
    fr = [f.clone().requires_grad_(True) for f in feats]
    fd = [f.to(_dev()).requires_grad_(True) for f in feats]
    sdg = _grad_sd(sd)
    cr, rr = O.head_forward(sdg, fr, cfg)
    cd, rd = m(fd)
    assert len(cd) == 5 and len(rd) == 5
    lr, l = 0, 0
    ftol = TOL_EXACT if prec == 'fp32' else 2e-4
    gtol = 5e-4 if prec == 'fp32' else 5e-2        # ReLU masks within round-off of zero flip (see note above)
    for a, b in list(zip(cd, cr)) + list(zip(rd, rr)):
        assert tuple(a.shape) == tuple(b.shape)
        assert _rel(a.detach().cpu(), b.detach()) < ftol
        wgt = torch.randn(b.shape, generator=g)
        lr = lr + (b * wgt).sum()
        l = l + (a * wgt.to(_dev())).sum()
    lr.backward()
    l.backward()
    for a, b in zip(fd, fr):
        assert _rel(a.grad.cpu(), b.grad) < gtol
    worst = _compare_param_grads(m, sdg, 'bbox_head.', tol=gtol)
    print('head', prec, 'worst grad rel err', worst)


@pytest.mark.parametrize('B,top', [(4, 32), (3, 64)])
def test_head_planes_path_forward_backward(B, top):
    """RetinaHead with the tower activations / gradients kept as bf16 hi/lo planes (conv_planes_kernel: TMA-fed im2col,
    epilogue writes the next layer's operand; weight gradients straight from the planes; bias gradients from the data
    gradients' column sums) against the CPU oracle: forward, feature gradients, every parameter gradient."""
    from models.retinahead import RetinaHead
    ops = _ops()
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    sd = O.init_state_dict(cfg, seed=33)
    m = _load(RetinaHead(num_classes=20, in_channels=64), sd, 'bbox_head.')
    g = torch.Generator().manual_seed(6)
    feats = [torch.randn(B, 64, top >> i, top >> i, generator=g) for i in range(5)]
    fr = [f.clone().requires_grad_(True) for f in feats]
    fd = [f.to(_dev()).requires_grad_(True) for f in feats]
    assert ops.head_planes_ok([ops.to_nhwc(f) for f in fd], m._params())          # this test is about the planes path
    sdg = _grad_sd(sd)
    cr, rr = O.head_forward(sdg, fr, cfg)
    cd, rd = m(fd)
    lr, l = 0, 0
    for a, b in list(zip(cd, cr)) + list(zip(rd, rr)):
        assert tuple(a.shape) == tuple(b.shape)
        assert _rel(a.detach().cpu(), b.detach()) < 2e-4
        wgt = torch.randn(b.shape, generator=g)
        lr = lr + (b * wgt).sum()
        l = l + (a * wgt.to(_dev())).sum()
    lr.backward()
    l.backward()
    errs = [_rel(a.grad.cpu(), b.grad) for a, b in zip(fd, fr)]
    worst = _compare_param_grads(m, sdg, 'bbox_head.', tol=5e-2)
    print('head planes path B=%d: feature grad rel errs %s, worst param grad %s' % (B, ['%.1e' % e for e in errs], worst))
    assert max(errs) < 5e-2


@pytest.mark.parametrize('K,B,top', [(3, 4, 32), (90, 2, 16), (1, 4, 32)])
def test_head_class_count_not_a_multiple_of_4(K, B, top):
    """The reference accepts any num_classes; the kernels move channels in vectors of 4, so RetinaHead pads every anchor's
    class block with zero-weight dummy classes (plain autograd ops around the fused head).  Forward, feature gradients
    and the gradients of the UNPADDED retina_cls parameters vs the CPU oracle; planes path (top=32, B=4) and the fallback."""
    from models.retinahead import RetinaHead
    cfg = O.make_config('efficientdet-d0', K, 64, 2)
    sd = O.init_state_dict(cfg, seed=35)
    m = _load(RetinaHead(num_classes=K, in_channels=64), sd, 'bbox_head.')
    assert tuple(m.retina_cls.weight.shape) == (9 * K, 256, 3, 3)
    g = torch.Generator().manual_seed(8)
    feats = [torch.randn(B, 64, top >> i, top >> i, generator=g) for i in range(5)]
    fr = [f.clone().requires_grad_(True) for f in feats]
    fd = [f.to(_dev()).requires_grad_(True) for f in feats]
    sdg = _grad_sd(sd)
    cr, rr = O.head_forward(sdg, fr, cfg)
    cd, rd = m(fd)
    lr, l = 0, 0
    for a, b in list(zip(cd, cr)) + list(zip(rd, rr)):
        assert tuple(a.shape) == tuple(b.shape)
        assert _rel(a.detach().cpu(), b.detach()) < 2e-4
        wgt = torch.randn(b.shape, generator=g)
        lr = lr + (b * wgt).sum()
        l = l + (a * wgt.to(_dev())).sum()
    lr.backward()
    l.backward()
    assert max(_rel(a.grad.cpu(), b.grad) for a, b in zip(fd, fr)) < 5e-2
    worst = _compare_param_grads(m, sdg, 'bbox_head.', tol=5e-2)
    print('head K=%d: worst param grad %s' % (K, worst))


def test_model_with_three_classes_train_step_and_inference():
    """Whole model with num_classes=3 (not a multiple of 4): train-step losses and gradients vs the oracle, then the
    inference path (decode + NMS) returns the oracle's detections."""
    K = 3
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=41)
    m = _build('efficientdet-d0', K, 64, 2, sd, is_training=True)
    m.eval()
    m.is_training = True
    images, ann = O.synthetic_batch(2, size=256, num_classes=K, seed=42)
    cl, rl = m([images.to(_dev()), ann.to(_dev())])
    (cl.mean() + rl.mean()).backward()
    sdg = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v) for k, v in sd.items()}
    ocl, orl = O.train_forward(sdg, images, ann, cfg)
    (ocl.mean() + orl.mean()).backward()
    assert _rel(cl.detach().cpu(), ocl.detach()) < 1e-3 and _rel(rl.detach().cpu(), orl.detach()) < 1e-3
    worst = 0.0
    for k, p in m.named_parameters():
        if sdg[k].grad is not None and float(sdg[k].grad.abs().max()) > 0:
            worst = max(worst, _rel(p.grad.cpu(), sdg[k].grad))
    assert worst < TOL_GRAD['bf16x3'], worst
    assert tuple(m.bbox_head.retina_cls.weight.grad.shape) == (9 * K, 256, 3, 3)
    m.is_training = False
    m.threshold = 0.03
    with torch.no_grad():
        det = m(images[:1].to(_dev()))
        ref = O.detect(sd, images[:1], cfg, threshold=0.03, iou_threshold=0.5)
    assert ref[0].numel() > 0 and abs(det[0].numel() - ref[0].numel()) <= max(3, ref[0].numel() // 20)


@pytest.mark.parametrize('empty_first', [False, True])
def test_focal_loss_forward_backward(empty_first):
    from models.losses import FocalLoss
    g = torch.Generator().manual_seed(7)
    B, K, size = 3, 20, 256
    anchors = torch.from_numpy(O.anchors_for(size, size))
    A = anchors.shape[1]
    cls = torch.rand(B, A, K, generator=g) * 0.2
    cls[0, :50] = 0.99995          # outside the clamp range -> zero gradient
    cls[1, :50] = 0.00002
    reg = torch.randn(B, A, 4, generator=g) * 0.3
    _, ann = O.synthetic_batch(B, size=size, num_classes=K, seed=9, empty_first=empty_first)
    ann[1, 7] = torch.tensor([10.0, 10.0, 10.4, 10.3, 3.0])   # sub-pixel box (width clamp branch)
    cr, rr = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    lc, lr = O.focal_loss(cr, rr, anchors, ann)
    (lc.mean() * 1.5 + lr.mean() * 0.5).backward()
    cd, rd = cls.to(_dev()).requires_grad_(True), reg.to(_dev()).requires_grad_(True)
    oc, orr = FocalLoss()(cd, rd, anchors.to(_dev()), ann.to(_dev()))
    assert tuple(oc.shape) == (1,) and tuple(orr.shape) == (1,)
    assert _rel(oc.detach().cpu(), lc.detach()) < TOL_EXACT
    assert _rel(orr.detach().cpu(), lr.detach()) < TOL_EXACT
    (oc.mean() * 1.5 + orr.mean() * 0.5).backward()
    assert _rel(cd.grad.cpu(), cr.grad) < TOL_EXACT
    assert _rel(rd.grad.cpu(), rr.grad) < TOL_EXACT


def test_anchors_bit_exact():
    from models.module import Anchors
    for (h, w) in [(512, 512), (256, 384), (1024, 1024)]:
        a = Anchors()(torch.zeros(1, 3, h, w, device=_dev()))
        assert torch.equal(a.cpu(), torch.from_numpy(O.anchors_for(h, w)))
    st = np.load(os.path.join(G, 'd0_512_fwd_wellcond.npz'))
    a = Anchors()(torch.zeros(1, 3, 512, 512, device=_dev())).cpu().numpy()
    import hashlib
    assert hashlib.sha256(a.tobytes()).digest() == bytes(st['anchors/sha256'])


# ------------------------------------------------------------------------------------------------
# whole model vs golden vectors of the real reference
# ------------------------------------------------------------------------------------------------

def _build(net, K, W, D, sd, is_training):
    from models import EfficientDet
    m = EfficientDet(num_classes=K, network=net, D_bifpn=D, W_bifpn=W, is_training=is_training)
    m.load_state_dict(sd)
    return m.to(_dev())


def _check_sampled(st, name, t, tol):
    s, i = st[name + '/s'], st[name + '/i']
    assert tuple(st[name + '/shape']) == tuple(t.shape), name
    got = t.detach().contiguous().view(-1).cpu()[torch.from_numpy(i)]
    e = _rel(got, torch.from_numpy(s))
    n = float(torch.linalg.vector_norm(t.detach().double()))
    assert abs(n - st[name + '/n'][0]) <= tol * max(st[name + '/n'][0], 1e-30), (name, n, st[name + '/n'][0])
    return e


@pytest.mark.parametrize('tag,net,W,D,K,mode', [
    ('d0_512_fwd_wellcond', 'efficientdet-d0', 64, 2, 80, 'wellcond'),
    ('d0_512_fwd_asbuilt', 'efficientdet-d0', 64, 2, 80, 'asbuilt'),
    ('d1_384_fwd_wellcond', 'efficientdet-d1', 88, 3, 20, 'wellcond'),
])
def test_model_forward_vs_reference_golden(tag, net, W, D, K, mode, prec):
    st = np.load(os.path.join(G, tag + '.npz'))
    seed, size, B = [int(v) for v in st['meta/seed']]
    cfg = O.make_config(net, num_classes=K, W_bifpn=W, D_bifpn=D)
    sd = O.init_state_dict(cfg, seed=seed, mode=mode)
    thr, iou = [float(v) for v in st['det/threshold']]
    m = _build(net, K, W, D, sd, is_training=False)
    m.threshold, m.iou_threshold = thr, iou
    m.eval()
    images, _ = O.synthetic_batch(B, size=size, seed=100 + seed)
    x = images[:1].to(_dev())
    with torch.no_grad():
        P = m.backbone(x)
        neck = m.neck(P[-5:])
        cls_l, reg_l = m.bbox_head(neck)
        det = m(x)
    worst = 0.0
    for li in range(7):
        worst = max(worst, _check_sampled(st, 'P%d' % li, P[li], TOL))
    for li in range(5):
        worst = max(worst, _check_sampled(st, 'bifpn%d_%d' % (D - 1, li), neck[li], TOL))
    cls, reg = torch.cat(cls_l, dim=1), torch.cat(reg_l, dim=1)
    worst = max(worst, _check_sampled(st, 'cls', cls, TOL), _check_sampled(st, 'reg', reg, TOL))
    print(tag, 'worst sampled rel err', worst)
    assert worst < TOL
    # detections: same count and same (score, class, box) rows up to fp32 round-off of the network
    # outputs; candidates whose score or IoU sits within round-off of a threshold may legitimately flip
    ref_s, ref_c, ref_b = st['det/scores'], st['det/classes'], st['det/boxes']
    assert det[1].dtype == torch.int64
    n_ref, n = ref_s.shape[0], det[0].numel()
    assert abs(n - n_ref) <= max(2, n_ref // 50), (n, n_ref)
    # order-insensitive row matching: near-equal scores may swap places, and a candidate within
    # round-off of a threshold may flip; everything else must agree row for row
    db, ds, dc = det[2].cpu().numpy(), det[0].cpu().numpy(), det[1].cpu().numpy()
    used, matched = np.zeros(n, dtype=bool), 0
    for j in range(n_ref):
        dist = np.abs(db - ref_b[j]).sum(axis=1) + used * 1e9
        i = int(np.argmin(dist))
        if dist[i] < (1e-2 if prec == 'fp32' else 0.5) and abs(ds[i] - ref_s[j]) < (1e-4 if prec == 'fp32' else 1e-3) \
                and dc[i] == ref_c[j]:
            used[i] = True
            matched += 1
    print(tag, 'detections matched %d / %d (ours %d)' % (matched, n_ref, n))
    if mode == 'asbuilt':
        # degenerate init: every score is 0.5 +- 1e-7, so the sort order / IoU chains are round-off noise
        assert matched >= 0.9 * n_ref
    else:
        assert matched >= n_ref - max(2, n_ref // 50)


@pytest.mark.parametrize('tag', ['d0_256_train_b2', 'd0_256_train_b2_empty'])
def test_model_train_step_vs_reference_golden(tag, prec):
    st = np.load(os.path.join(G, tag + '.npz'))
    seed, size, B, empty = [int(v) for v in st['meta/seed']]
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=seed, mode='wellcond')
    m = _build('efficientdet-d0', 20, 64, 2, sd, is_training=True)
    m.eval()
    m.is_training = True
    images, ann = O.synthetic_batch(B, size=size, num_classes=20, seed=200 + seed, empty_first=bool(empty))
    cl, rl = m([images.to(_dev()), ann.to(_dev())])
    assert tuple(cl.shape) == (1,) and tuple(rl.shape) == (1,)
    assert _rel(cl.detach().cpu(), torch.from_numpy(st['loss/cls'])) < TOL
    assert _rel(rl.detach().cpu(), torch.from_numpy(st['loss/reg'])) < TOL
    (cl.mean() + rl.mean()).backward()
    params = dict(m.named_parameters())
    names, norms = [str(k) for k in st['grad_names']], st['grad_norms']
    worst = (0.0, None)
    for k, n in zip(names, norms):
        g = params[k].grad
        assert g is not None, k
        gn = float(torch.linalg.vector_norm(g.double()))
        e = abs(gn - n) / max(n, 1e-30)
        key = 'grad/' + k
        if key in st.files:
            e = max(e, _rel(g.cpu(), torch.from_numpy(st[key])))
        elif ('gsamp/' + k + '/s') in st.files:
            idx = torch.from_numpy(st['gsamp/' + k + '/i'])
            e = max(e, _rel(g.detach().cpu().view(-1)[idx], torch.from_numpy(st['gsamp/' + k + '/s'])))
        if e > worst[0]:
            worst = (e, k)
        assert e < TOL_GRAD[prec], (k, e)
    print(tag, prec, 'worst grad rel err', worst)
    for k in ('backbone._conv_head.weight', 'backbone._bn1.weight', 'backbone._fc.weight'):
        assert params[k].grad is None


def test_d0_512_train_mode_step_vs_oracle(prec):
    """The mode bench.py times (reference train.py:100-102): model.train(); freeze_bn() -> drop-connect ACTIVE,
    BatchNorm frozen, D0 at 512x512, B=4.  The CUDA torch.rand([B,1,1,1]) stream the product consumes (one draw per
    skip block, models/utils.py:79-90) is replayed into the oracle, so forward AND backward of the drop-connect
    path (row_scale in the project-conv epilogue and in the BN2 backward) are parity-checked: losses <= 1e-3,
    every parameter gradient within TOL_GRAD."""
    B = 4
    cfg = O.make_config('efficientdet-d0', num_classes=80, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=0)
    m = _build('efficientdet-d0', 80, 64, 2, sd, is_training=True)
    m.train()
    m.is_training = True
    m.freeze_bn()
    images, ann = O.synthetic_batch(B, size=512, num_classes=80, seed=1000)
    torch.manual_seed(4321)
    cl, rl = m([images.to(_dev()), ann.to(_dev())])
    (cl.mean() + rl.mean()).backward()
    torch.manual_seed(4321)
    nskip = sum(1 for i, b in enumerate(cfg['blocks']) if b['skip'] and i > 0)
    keeps = [torch.rand([B, 1, 1, 1], dtype=torch.float32, device=_dev()).cpu() for _ in range(nskip)]
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    sdg = _grad_sd(sd)
    ocl, orl = O.train_forward(sdg, images, ann, cfg, keep_samples=keeps)
    (ocl.mean() + orl.mean()).backward()
    e_c, e_r = _rel(cl.detach().cpu(), ocl.detach()), _rel(rl.detach().cpu(), orl.detach())
    assert e_c < TOL and e_r < TOL, (e_c, e_r)
    worst = _compare_param_grads(m, sdg, '', tol=TOL_GRAD[prec])
    print('d0 512 train mode', prec, 'losses', float(cl), float(rl), 'rel', e_c, e_r, 'worst grad', worst,
          'keep draws', len(keeps))


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs[3] / configs[4]: the larger family members as parity cases (oracle on the host)
# ------------------------------------------------------------------------------------------------

def test_d4_1024_train_step_vs_oracle():
    """EfficientDet-D4 geometry (B4 backbone, W_bifpn 224, D_bifpn 6 per utils/config_eff.py, 1024x1024):
    one forward+backward, losses and a spread of parameter gradients against the CPU oracle."""
    cfg = O.make_config('efficientdet-d4', num_classes=20, W_bifpn=224, D_bifpn=6)
    sd = O.init_state_dict(cfg, seed=41)
    m = _build('efficientdet-d4', 20, 224, 6, sd, is_training=True)
    m.eval()
    m.is_training = True
    images, ann = O.synthetic_batch(1, size=1024, num_classes=20, seed=42)
    cl, rl = m([images.to(_dev()), ann.to(_dev())])
    (cl.mean() + rl.mean()).backward()
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    sdg = _grad_sd(sd)
    ocl, orl = O.train_forward(sdg, images, ann, cfg)
    (ocl.mean() + orl.mean()).backward()
    assert _rel(cl.detach().cpu(), ocl.detach()) < TOL and _rel(rl.detach().cpu(), orl.detach()) < TOL
    params = dict(m.named_parameters())
    worst = (0.0, None)
    for k, p in params.items():
        ref = sdg[k].grad
        if ref is None or float(ref.abs().max()) == 0.0:
            continue
        e = _rel(p.grad.cpu(), ref)
        if e > worst[0]:
            worst = (e, k)
    print('d4 1024 losses', float(cl), float(rl), 'worst grad rel err', worst)
    assert worst[0] < TOL_GRAD['bf16x3']


def test_d7_1536_inference_vs_oracle():
    """EfficientDet-D7 geometry (B6 backbone, W_bifpn 384, D_bifpn 8, 1536x1536, 441 936 anchors):
    forward + decode + NMS on the device against the CPU oracle."""
    cfg = O.make_config('efficientdet-d7', num_classes=20, W_bifpn=384, D_bifpn=8)
    sd = O.init_state_dict(cfg, seed=51)
    m = _build('efficientdet-d7', 20, 384, 8, sd, is_training=False)
    m.eval()
    images, _ = O.synthetic_batch(1, size=1536, seed=52)
    x = images.to(_dev())
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    with torch.no_grad():
        ocls, oreg, _ = O.raw_outputs(sd, images, cfg)
    # eval.py:349-352 uses 0.4; with random weights pick the score of the ~6000th best anchor instead so the
    # (quadratic, numpy) oracle NMS stays affordable -- both sides get the same threshold
    thr = float(torch.sort(ocls.max(dim=2)[0].flatten(), descending=True)[0][6000])
    thr = max(thr, 0.05)
    m.threshold, m.iou_threshold = thr, 0.5
    with torch.no_grad():
        feats = m.extract_feat(x)
        cls_l, reg_l = m.bbox_head(feats)
        det = m(x)
    coll = {}
    with torch.no_grad():
        ref = O.detect(sd, images, cfg, threshold=thr, iou_threshold=0.5, collect=coll)
    cls, reg = torch.cat(cls_l, dim=1), torch.cat(reg_l, dim=1)
    assert cls.shape[1] == 441936
    e_c, e_r = _rel(cls.cpu(), coll['cls']), _rel(reg.cpu(), coll['reg'])
    print('d7 1536: cls rel %.2e reg rel %.2e, detections ours %d oracle %d' % (e_c, e_r, det[0].numel(), ref[0].numel()))
    assert e_c < TOL and e_r < TOL
    n_ref = ref[0].numel()
    assert abs(det[0].numel() - n_ref) <= max(3, n_ref // 25)


# ------------------------------------------------------------------------------------------------
# SURVEY 8(f) rank 1: fused clip_grad_norm_ + AdamW vs torch's own implementations on the CPU
# ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('max_norm', [0.1, 1e9])
def test_fused_clip_adamw_matches_torch(max_norm):
    from models.fused_optim import FusedClipAdamW
    g = torch.Generator().manual_seed(3)
    shapes = [(1,), (7,), (33, 31), (256, 64, 3, 3), (65537,), (300001,), (16,)]
    ref_p = [torch.nn.Parameter(torch.randn(s, generator=g)) for s in shapes]
    dev_p = [torch.nn.Parameter(p.detach().clone().to(_dev())) for p in ref_p]
    extra_ref = torch.nn.Parameter(torch.randn(5, generator=g))          # never receives a gradient (dead parameter)
    extra_dev = torch.nn.Parameter(extra_ref.detach().clone().to(_dev()))
    ref_opt = torch.optim.AdamW(ref_p + [extra_ref], lr=1e-2)
    dev_opt = FusedClipAdamW(dev_p + [extra_dev], lr=1e-2, max_norm=max_norm)
    for it in range(3):
        for a, b in zip(ref_p, dev_p):
            grad = torch.randn(a.shape, generator=g) * (0.5 + it)
            a.grad = grad.clone()
            b.grad = grad.clone().to(_dev())
        total = torch.nn.utils.clip_grad_norm_(ref_p + [extra_ref], max_norm)
        ref_opt.step()
        dev_opt.step()
        assert abs(float(dev_opt.last_norm_sq.sqrt()) - float(total)) <= 1e-5 * float(total)
        for a, b in zip(ref_p, dev_p):
            assert _rel(b.grad.cpu(), a.grad) < 5e-6          # gradients rescaled in place like clip_grad_norm_
            assert _rel(b.detach().cpu(), a.detach()) < 5e-6, it
    assert torch.equal(extra_dev.detach().cpu(), extra_ref.detach())


# ------------------------------------------------------------------------------------------------
# SURVEY 8(f) rank 3: batched inference = the reference's single-image post-processing applied per image
# ------------------------------------------------------------------------------------------------

def _match_rows(det, ref, tol_box, tol_score):
    """order-insensitive count of reference detections (score, class, box) found in det"""
    s, c, b = det
    rs, rc, rb = ref
    used, matched = np.zeros(s.shape[0], dtype=bool), 0
    for j in range(rs.shape[0]):
        dist = np.abs(b - rb[j]).sum(axis=1) + used * 1e9
        k = int(np.argmin(dist)) if s.shape[0] else -1
        if k >= 0 and dist[k] < tol_box and abs(s[k] - rs[j]) < tol_score and c[k] == rc[j]:
            used[k] = True
            matched += 1
    return matched


def test_detect_batch_matches_per_image_reference(prec):
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=61)
    m = _build('efficientdet-d0', 20, 64, 2, sd, is_training=False)
    m.eval()
    images, _ = O.synthetic_batch(3, size=256, seed=62)
    with torch.no_grad():
        ocls, _, _ = O.raw_outputs(sd, images, cfg)
    thr = float(torch.sort(ocls.max(dim=2)[0][0], descending=True)[0][400])
    m.threshold, m.iou_threshold = thr, 0.5
    x = images.to(_dev())
    dets = m.detect_batch(x)
    with torch.no_grad():
        first = m(x)                                   # the reference API: image 0 of the same batch
    assert len(dets) == 3
    tol_box, tol_score = (1e-2, 1e-4) if prec == 'fp32' else (0.5, 1e-3)
    # two passes over the same batch differ only by the order of the fp32 atomics of the SE mean
    d0 = [t.cpu().numpy() for t in dets[0]]
    f0 = [t.cpu().numpy() for t in first]
    assert abs(d0[0].shape[0] - f0[0].shape[0]) <= 1
    assert _match_rows(d0, f0, 1e-2, 1e-4) >= f0[0].shape[0] - 1
    for i in range(3):
        with torch.no_grad():
            ref = [t.numpy() for t in O.detect(sd, images[i:i + 1], cfg, threshold=thr, iou_threshold=0.5)]
        det = [t.cpu().numpy() for t in dets[i]]
        assert dets[i][1].dtype == torch.int64 and det[2].shape[1:] == (4,)
        n_ref, n = ref[0].shape[0], det[0].shape[0]
        assert n_ref > 20 and abs(n - n_ref) <= 2, (i, n, n_ref)
        matched = _match_rows(det, ref, tol_box, tol_score)
        print('image', i, 'matched %d / %d (ours %d)' % (matched, n_ref, n))
        assert matched >= n_ref - 2, (i, matched, n_ref)
    # nothing above the threshold -> empty triples, as forward() returns for image 0
    m.threshold = 2.0
    for trip in m.detect_batch(x):
        assert trip[0].numel() == 0 and trip[1].numel() == 0 and tuple(trip[2].shape) == (0, 4)


def test_data_edits_are_seen_after_invalidate_caches():
    """ADVICE r1: in-place writes through `.data` do not bump Tensor._version, so the packed-weight cache would keep
    serving the old weights; invalidate_caches() (called by load_state_dict / train / eval / freeze_bn) fixes that."""
    ops = _ops()
    from models.module import ConvModule
    conv = ConvModule(8, 16, 3, padding=1, activation=None).to(_dev())
    x = torch.randn(1, 8, 8, 8, device=_dev())
    y0 = conv(x).clone()
    v0 = conv.conv.weight._version
    conv.conv.weight.data.mul_(2.0)                          # invisible to the version counter
    assert conv.conv.weight._version == v0
    ops.invalidate_caches()
    y1 = conv(x)
    b = conv.conv.bias.detach().view(1, -1, 1, 1)
    assert _rel((y1 - b).cpu(), (2.0 * (y0 - b)).cpu()) < 1e-5


def test_checkpoint_save_resume_round_trip(tmp_path):
    """SURVEY.md 8(f) rank 4 (train.py:213-236,279-291): train 2 steps with the fused optimizer, save model + optimizer
    state the way train.py does under DDP (keys prefixed `module.`), resume in a fresh model / optimizer, take the
    third step on both: parameters must agree (fp32 atomics order is the only difference)."""
    from models.fused_optim import FusedClipAdamW
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=9)
    images, ann = O.synthetic_batch(2, size=128, num_classes=20, seed=10)
    images, ann = images.to(_dev()), ann.to(_dev())

    def make():
        m = _build('efficientdet-d0', 20, 64, 2, sd, is_training=True)
        m.eval()
        m.is_training = True
        return m, FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)

    def step(m, opt):
        opt.zero_grad()
        cl, rl = m([images, ann])
        (cl.mean() + rl.mean()).backward()
        opt.step()

    a, opt_a = make()
    step(a, opt_a)
    step(a, opt_a)
    path = os.path.join(tmp_path, 'ckpt.pth')
    torch.save({'state_dict': {'module.' + k: v for k, v in a.state_dict().items()}, 'optimizer': opt_a.state_dict()}, path)
    ck = torch.load(path, map_location='cpu')
    b, opt_b = make()
    b.load_state_dict(ck['state_dict'])
    opt_b.load_state_dict(ck['optimizer'])
    for (k, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(pa, pb), k
    step(a, opt_a)
    step(b, opt_b)
    worst = max(_rel(pb, pa) for pa, pb in zip(a.parameters(), b.parameters()))
    assert worst < 2e-4, worst        # one more optimizer step each; fp32 atomics order differs between the two runs
    assert int(opt_b.state[next(iter(b.parameters()))]['step']) == 3


def test_graphed_train_step_equals_eager():
    """models/graph_step.py: the captured step (forward + loss + backward as one CUDA graph) reproduces the eager step
    on new inputs copied into its static buffers: same loss, same gradients (fp32 atomics order aside)."""
    from models.graph_step import GraphedTrainStep
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=13)
    m = _build('efficientdet-d0', 20, 64, 2, sd, is_training=True)
    m.eval()                                                  # drop-connect off: eager and replay must see the same function
    m.is_training = True
    batches = [O.synthetic_batch(2, size=256, num_classes=20, seed=s_) for s_ in (20, 21)]
    eager = []
    for images, ann in batches:
        for p in m.parameters():
            p.grad = None
        cl, rl = m([images.to(_dev()), ann.to(_dev())])
        (cl.mean() + rl.mean()).backward()
        eager.append((float(cl + rl), {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}))
    del cl, rl                                                # a live eager graph pins the grad accumulators to the legacy stream
    step = GraphedTrainStep(m, batches[0][0].to(_dev()), batches[0][1].to(_dev()))
    for (images, ann), (loss_e, grads_e) in zip(batches, eager):
        loss = step(images.to(_dev()), ann.to(_dev()))
        torch.cuda.synchronize()
        assert abs(float(loss) - loss_e) <= 1e-4 * abs(loss_e)
        errs = sorted(_rel(p.grad, grads_e[k]) for k, p in m.named_parameters() if k in grads_e and float(grads_e[k].abs().max()) > 0)
        # same kernels, same inputs: only the order of the fp32 atomics differs between two runs, amplified by the
        # network's gradient conditioning on a few parameters (tools/grad_conditioning.py) -- 6e-3 worst seen
        assert errs[len(errs) // 2] < 1e-3 and errs[-1] < TOL_GRAD['bf16x3'], (errs[len(errs) // 2], errs[-1])
