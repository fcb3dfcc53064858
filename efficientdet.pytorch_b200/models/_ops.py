"""Host-side glue between the nn.Module mirror and the C ABI: tensor allocation, parameter-derived
caches (packed weights, folded BatchNorm) and the ``torch.autograd.Function``s whose forward /
backward are sequences of ``libeffdet_b200.so`` launches.  No arithmetic happens in PyTorch here
(torch only allocates, zero-fills and takes views); gradients come back as ordinary ``.grad``
so DDP's reducer hooks and ``clip_grad_norm_`` (reference train.py:114-116) keep working.

Internal activation layout is NHWC fp32; module boundaries expose the same memory as a logical
NCHW tensor with channels_last strides (zero-copy ``permute`` views).
"""
import collections
import os
import weakref

import torch

from . import _native as N
from ._native import ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SWISH, FUSE_POOL, FUSE_UP

# ------------------------------------------------------------------------------------------------
# layout helpers
# ------------------------------------------------------------------------------------------------


class _ToNHWC(torch.autograd.Function):
    """NCHW-contiguous -> NHWC-contiguous through the library's tiled transpose."""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        B, C, H, W = x.shape
        y = torch.empty((B, H, W, C), device=x.device, dtype=torch.float32)
        N.call('effdet_nchw_to_nhwc', x, N.f32(x, 'x'), N.f32(y), B, C, H, W)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        B, H, W, C = dy.shape
        dx = torch.empty((B, C, H, W), device=dy.device, dtype=torch.float32)
        N.call('effdet_nhwc_to_nchw', dy, N.f32(dy), N.f32(dx), B, C, H, W)
        return dx


def check_cuda_f32(x, what):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise N.EffdetNativeError('%s: expected a CUDA tensor; the H100 hot path has no CPU fallback '
                                  '(got %s)' % (what, getattr(x, 'device', type(x))))
    if x.dtype != torch.float32:
        raise N.EffdetNativeError('%s: expected float32, got %s' % (what, x.dtype))


def to_nhwc(x, what='input'):
    """Logical NCHW tensor -> NHWC-contiguous tensor (zero-copy when already channels_last)."""
    check_cuda_f32(x, what)
    if x.dim() != 4:
        raise N.EffdetNativeError('%s: expected a 4-D NCHW tensor, got shape %s' % (what, tuple(x.shape)))
    v = x.permute(0, 2, 3, 1)
    if v.is_contiguous():
        return v
    return _ToNHWC.apply(x)


def to_nchw_view(y):
    """NHWC-contiguous tensor -> logical NCHW view (channels_last strides, zero-copy)."""
    return y.permute(0, 3, 1, 2)


def _empty(shape, like):
    return torch.empty(shape, device=like.device, dtype=torch.float32)


def _zeros(shape, like):
    return torch.zeros(shape, device=like.device, dtype=torch.float32)


def _zeros_like_many(tensors):
    """Zero-initialised gradient buffers for `tensors` carved out of ONE allocation / ONE memset (each
    slice 16-byte aligned) instead of one fill kernel per parameter."""
    sizes = [(t.numel() + 3) // 4 * 4 for t in tensors]
    flat = torch.zeros((sum(sizes),), device=tensors[0].device, dtype=torch.float32)
    out, off = [], 0
    for t, n in zip(tensors, sizes):
        out.append(flat[off:off + t.numel()].view(t.shape))
        off += n
    return out


def _stash(ctx, name):
    """Activations a fused node keeps for its backward live on ctx and are released by the first backward (the step's
    activation memory must not outlive it).  A second backward (retain_graph=True) therefore cannot be served."""
    v = getattr(ctx, name)
    if v is None:
        raise N.EffdetNativeError('backward was called a second time on a fused EfficientDet node: its saved activations are '
                                  'released after the first backward (retain_graph=True is not supported; run forward again)')
    return v


# ------------------------------------------------------------------------------------------------
# parameter-derived caches (invalidated by in-place updates: optimizer.step, load_state_dict)
# ------------------------------------------------------------------------------------------------
_cache = {}   # id(first tensor) -> (weakref to it, {kind: (signature, value)})


def invalidate_caches():
    """Drop every packed weight / folded BatchNorm derived from parameters.  The caches are keyed on
    (Tensor._version, data_ptr), which in-place writes through `.data` (`w.data.normal_()`, the idiom the reference's
    own __init__ uses, models/efficientdet.py:47-53; EMA swaps `p.data.copy_()`) do NOT bump: after such an edit call
    this (EfficientDet.load_state_dict / train / eval / freeze_bn do it for you)."""
    _cache.clear()


def _cached(params, kind, builder):
    key_t = params[0]
    kid = id(key_t)
    sig = tuple((p._version, p.data_ptr()) for p in params)
    ent = _cache.get(kid)
    if ent is None or ent[0]() is not key_t:
        ent = (weakref.ref(key_t, lambda _r, kid=kid: _cache.pop(kid, None)), {})
        _cache[kid] = ent
    hit = ent[1].get(kind)
    if hit is not None and hit[0] == sig:
        return hit[1]
    val = builder()
    ent[1][kind] = (sig, val)
    return val


def pack_conv(w):
    """OIHW parameter -> (forward pack [kk][Cin][Cout], dgrad pack [kk][Cout][Cin])."""
    def build():
        Cout, Cin, k, _ = w.shape
        src = w.detach().contiguous()
        wf = _empty((k * k, Cin, Cout), w)
        wd = _empty((k * k, Cout, Cin), w)
        N.call('effdet_pack_conv_weight', w, N.f32(src, 'conv weight'), N.f32(wf), N.f32(wd), Cout, Cin, k)
        return wf, wd
    return _cached([w], 'pack', build)


# Precision of the dense 1x1 / 3x3 convolutions of neck and head (95 % of the FLOPs):
#   'bf16x3' (default): wgmma tensor cores, operands split into bf16 hi+lo, three MMAs per product
#                       (~2^-16 relative per product, fp32 accumulation)
#   'bf16'            : the same routing, but the dense 3x3 convs (BiFPN nodes, head towers, class / box convs; forward,
#                       data and weight gradient) take one MMA per product: bf16-rounded operands, fp32 accumulation.
#                       The 1x1 convs stay on bf16x3 (they are HBM-bound, a single pass would buy no time)
#   'fp32'            : exact fp32 FMA on the CUDA cores
PRECISION = os.environ.get('EFFDET_B200_PRECISION', 'bf16x3')


def tc_enabled():
    """route the dense convs to the tensor cores (bf16x3 or bf16 mode)"""
    return PRECISION in ('bf16x3', 'bf16')


def tc_single(k):
    """1 when a k x k tensor-core conv takes one bf16 product per multiply-add (bf16 mode, 3x3 only), else 0"""
    return 1 if PRECISION == 'bf16' and k == 3 else 0


def pack_conv_tc(w):
    """OIHW parameter -> (forward, dgrad) pre-split bf16 hi/lo planes for the tensor-core kernels."""
    def build():
        Cout, Cin, k, _ = w.shape
        lib = N.load()
        kin, kout = lib.effdet_conv_tc_kpad(Cin), lib.effdet_conv_tc_kpad(Cout)
        src = w.detach().contiguous()
        tf = torch.empty((2, Cout, k * k, kin), device=w.device, dtype=torch.bfloat16)
        td = torch.empty((2, Cin, k * k, kout), device=w.device, dtype=torch.bfloat16)
        N.call('effdet_pack_conv_weight_tc', w, N.f32(src, 'conv weight'), tf.data_ptr(), td.data_ptr(), Cout, Cin, k)
        return tf, td
    return _cached([w], 'packtc', build)


def tc_packs(w):
    """(fwd, dgrad) tensor-core packs, or (None, None) when the fp32 path is selected / unsupported."""
    if not tc_enabled() or w.shape[0] % 4 or w.shape[1] % 4 or w.shape[0] < 16:
        return None, None
    return pack_conv_tc(w)


def pack_dw(w):
    """[C,1,k,k] depthwise parameter -> [k][k][C]."""
    def build():
        C, _, k, _ = w.shape
        src = w.detach().contiguous()
        o = _empty((k, k, C), w)
        N.call('effdet_pack_dw_weight', w, N.f32(src, 'depthwise weight'), N.f32(o), C, k)
        return o
    return _cached([w], 'packdw', build)


def bn_fold(gamma, beta, rmean, rvar, eps):
    """Frozen BN -> (scale, shift, rstd), each [C]."""
    def build():
        C = gamma.numel()
        scale, shift, rstd = _empty((C,), gamma), _empty((C,), gamma), _empty((C,), gamma)
        N.call('effdet_bn_fold', gamma, N.f32(gamma.detach(), 'bn weight'), N.f32(beta.detach(), 'bn bias'),
               N.f32(rmean, 'running_mean'), N.f32(rvar, 'running_var'), float(eps), N.f32(scale), N.f32(shift),
               N.f32(rstd), C)
        return scale, shift, rstd
    return _cached([gamma, beta, rmean, rvar], 'fold', build)


# ------------------------------------------------------------------------------------------------
# thin wrappers over single entry points
# ------------------------------------------------------------------------------------------------


def conv2d_raw(dev_t, x_ptr, x_bs, wf, y_ptr, y_bs, B, H, W, Cin, Cout, k, z_ptr=None, bias=None, scale=None,
               shift=None, a_scale=None, row_scale=None, res_ptr=None, res_bs=0, mask_ptr=None, mask_bs=0,
               act=ACT_NONE, w_tc=None, in_scale=None, in_shift=None, x_planes=None):
    a = N.ConvArgs(x_ptr, x_bs, N.f32(wf, 'packed weight'), y_ptr, y_bs, z_ptr, N.f32(bias, 'bias'),
                   N.f32(scale, 'scale'), N.f32(shift, 'shift'), N.f32(a_scale, 'a_scale'),
                   N.f32(row_scale, 'row_scale'), res_ptr, res_bs, mask_ptr, mask_bs, B, H, W, Cin, Cout, k, act,
                   w_tc.data_ptr() if w_tc is not None else None, N.f32(in_scale, 'in_scale'),
                   N.f32(in_shift, 'in_shift'), N.ptr(x_planes), tc_single(k) if w_tc is not None else 0)
    N.call('effdet_conv2d', dev_t, a)


def split_planes_like(x):
    """bf16 hi/lo plane buffer [2, B, H, W, C] for an NHWC fp32 tensor shape (x ~= hi + lo, the tensor-core operand form)."""
    return torch.empty((2,) + tuple(x.shape), device=x.device, dtype=torch.bfloat16)


def conv2d_from_planes(planes, wf, Cout, residual=None, w_tc=None):
    """1x1 conv whose input exists only as bf16 hi/lo planes [2,B,H,W,Cin] (written by effdet_dwconv_bwd_fused)."""
    _, B, H, W, Cin = planes.shape
    y = torch.empty((B, H, W, Cout), device=planes.device, dtype=torch.float32)
    bs = H * W * Cout
    conv2d_raw(y, None, H * W * Cin, wf, N.f32(y), bs, B, H, W, Cin, Cout, 1, res_ptr=N.f32(residual, 'residual'), res_bs=bs,
               w_tc=w_tc, x_planes=planes)
    return y


def conv2d(x, wf, Cout, k, bias=None, scale=None, shift=None, a_scale=None, row_scale=None, residual=None,
           mask_src=None, act=ACT_NONE, save_z=False, w_tc=None, in_scale=None, in_shift=None):
    """x NHWC contiguous -> y NHWC (and the raw pre-affine z when save_z).  in_scale/in_shift: x is a raw conv
    output and the operand is swish(x*in_scale+in_shift), applied while the tile is staged."""
    B, H, W, Cin = x.shape
    y = _empty((B, H, W, Cout), x)
    z = _empty((B, H, W, Cout), x) if save_z else None
    bs = H * W * Cout
    conv2d_raw(x, N.f32(x, 'x'), H * W * Cin, wf, N.f32(y), bs, B, H, W, Cin, Cout, k, z_ptr=N.f32(z), bias=bias,
               scale=scale, shift=shift, a_scale=a_scale, row_scale=row_scale, res_ptr=N.f32(residual, 'residual'),
               res_bs=bs, mask_ptr=N.f32(mask_src, 'mask_src'), mask_bs=bs, act=act, w_tc=w_tc, in_scale=in_scale,
               in_shift=in_shift)
    return (y, z) if save_z else y


def conv2d_multi_raw(dev_t, levels, wf, Cin, Cout, k, bias=None, act=ACT_NONE, w_tc=None):
    """One launch over several feature maps that share weights.  levels: dicts with x_ptr, x_bs, y_ptr, y_bs,
    B, H, W and optional res_ptr/res_bs, mask_ptr/mask_bs."""
    nl = len(levels)
    arr = (N.ConvArgs * nl)()
    wfp, bp = N.f32(wf, 'packed weight'), N.f32(bias, 'bias')
    tcp = w_tc.data_ptr() if w_tc is not None else None
    single = tc_single(k) if w_tc is not None else 0
    for i, lv in enumerate(levels):
        arr[i] = N.ConvArgs(lv['x_ptr'], lv['x_bs'], wfp, lv['y_ptr'], lv['y_bs'], None, bp, None, None, None, None,
                            lv.get('res_ptr'), lv.get('res_bs', 0), lv.get('mask_ptr'), lv.get('mask_bs', 0),
                            lv['B'], lv['H'], lv['W'], Cin, Cout, k, act, tcp, tc_single=single)
    N.call('effdet_conv2d_multi', dev_t, arr, nl)


def conv2d_multi(xs, wf, Cout, k, bias=None, act=ACT_NONE, w_tc=None, residuals=None, masks=None):
    """xs: list of NHWC tensors (same channel count) -> list of NHWC outputs, one kernel launch."""
    ys, levels = [], []
    for i, x in enumerate(xs):
        B, H, W, Cin = x.shape
        y = _empty((B, H, W, Cout), x)
        ys.append(y)
        lv = dict(x_ptr=N.f32(x, 'x'), x_bs=H * W * Cin, y_ptr=N.f32(y), y_bs=H * W * Cout, B=B, H=H, W=W)
        if residuals is not None and residuals[i] is not None:
            lv.update(res_ptr=N.f32(residuals[i], 'residual'), res_bs=H * W * Cout)
        if masks is not None and masks[i] is not None:
            lv.update(mask_ptr=N.f32(masks[i], 'mask_src'), mask_bs=H * W * Cout)
        levels.append(lv)
    conv2d_multi_raw(xs[0], levels, wf, xs[0].shape[3], Cout, k, bias=bias, act=act, w_tc=w_tc)
    return ys


def _ws_dw(dev_t, Cin, Cout, k):
    """the fp32 [9][Cout][Cin] workspace a 3x3 tensor-core weight gradient reduces into (1x1: None, dw itself)"""
    return torch.empty((9 * Cout * Cin,), device=dev_t.device, dtype=torch.float32) if k == 3 else None


def conv_wgrad_raw(dev_t, x_ptr, x_bs, dy_ptr, dy_bs, dw, dbias, B, H, W, Cin, Cout, k, a_scale=None, tc=False,
                   in_scale=None, in_shift=None, dy_planes=None):
    ws_x = ws_dy = ws_dw = None
    if tc:
        ws_dw = _ws_dw(dev_t, Cin, Cout, k)
        lib = N.load()
        ws_x = torch.empty((2 * B * H * W * lib.effdet_conv_tc_kpad(Cin),), device=dev_t.device, dtype=torch.bfloat16)
        if dy_planes is None:
            ws_dy = torch.empty((2 * B * H * W * lib.effdet_conv_tc_kpad(Cout),), device=dev_t.device, dtype=torch.bfloat16)
    a = N.WgradArgs(x_ptr, x_bs, dy_ptr, dy_bs, N.f32(dw, 'dw'), N.f32(dbias, 'dbias'), N.f32(a_scale, 'a_scale'),
                    B, H, W, Cin, Cout, k, 1 if tc else 0, ws_x.data_ptr() if ws_x is not None else None,
                    ws_dy.data_ptr() if ws_dy is not None else None, N.f32(in_scale, 'in_scale'),
                    N.f32(in_shift, 'in_shift'), N.ptr(dy_planes), None, tc_single(k) if tc else 0,
                    ws_dw.data_ptr() if ws_dw is not None else None)
    N.call('effdet_conv2d_wgrad', dev_t, a)


def pixel_boxes_ok(maps):
    """do the TMA-fed tensor-core kernels find a pixel box for every map?  maps: (B, H, W, ...) shapes"""
    lib = N.load()
    return all(lib.effdet_wgrad_tc_geometry_ok(m[0], m[1], m[2]) for m in maps)


def planes_ok(B, H, W, C):
    """can a [B,H,W,C] gradient be handed to the tensor-core weight / data gradients as bf16 hi/lo planes?"""
    return tc_enabled() and C % 8 == 0 and pixel_boxes_ok([(B, H, W)])


def conv_wgrad_multi(dev_t, levels, dw, dbias, Cin, Cout, k, tc=False):
    """Weight gradient of one shared-weight layer over several feature maps, accumulated into dw/dbias by ONE
    launch.  levels: dicts with x_ptr, x_bs, dy_ptr, dy_bs, B, H, W."""
    nl = len(levels)
    arr = (N.WgradArgs * nl)()
    keep = []
    lib = N.load()
    kin, kout = lib.effdet_conv_tc_kpad(Cin), lib.effdet_conv_tc_kpad(Cout)
    ws_dw = _ws_dw(dev_t, Cin, Cout, k) if tc else None
    for i, lv in enumerate(levels):
        ws_x = ws_dy = None
        if tc:
            npx = lv['B'] * lv['H'] * lv['W']
            ws_x = torch.empty((2 * npx * kin,), device=dev_t.device, dtype=torch.bfloat16)
            ws_dy = torch.empty((2 * npx * kout,), device=dev_t.device, dtype=torch.bfloat16)
            keep += [ws_x, ws_dy]
        arr[i] = N.WgradArgs(lv['x_ptr'], lv['x_bs'], lv['dy_ptr'], lv['dy_bs'], N.f32(dw, 'dw'), N.f32(dbias, 'dbias'),
                             None, lv['B'], lv['H'], lv['W'], Cin, Cout, k, 1 if tc else 0,
                             ws_x.data_ptr() if ws_x is not None else None, ws_dy.data_ptr() if ws_dy is not None else None,
                             tc_single=tc_single(k) if tc else 0, ws_dw=ws_dw.data_ptr() if ws_dw is not None else None)
    N.call('effdet_conv2d_wgrad_multi', dev_t, arr, nl)


def conv_wgrad(x, dy, dw, dbias, k, a_scale=None, tc=False, in_scale=None, in_shift=None):
    B, H, W, Cin = x.shape
    Cout = dy.shape[3]
    conv_wgrad_raw(x, N.f32(x, 'x'), H * W * Cin, N.f32(dy, 'dy'), H * W * Cout, dw, dbias, B, H, W, Cin, Cout, k,
                   a_scale=a_scale, tc=tc, in_scale=in_scale, in_shift=in_shift)


def bnact_bwd(dy, z, scale, shift, mean, rstd, act, row_scale=None, gate=None, dmean=None):
    """-> (dz, dgamma, dbeta) for y = act(z*scale+shift) [* row_scale]; SE mode when gate is given."""
    B = z.shape[0]
    C = z.shape[-1]
    HW = z.numel() // (B * C)
    dz = torch.empty_like(z)
    gb = _zeros((2 * C,), z)
    dgamma, dbeta = gb[:C], gb[C:]
    a = N.BnActBwdArgs(N.f32(dy, 'dy'), N.f32(z, 'z'), N.f32(dz), N.f32(scale), N.f32(shift), N.f32(mean, 'mean'),
                       N.f32(rstd), N.f32(dgamma), N.f32(dbeta), N.f32(row_scale), N.f32(gate), N.f32(dmean),
                       1.0 / HW, B, HW, C, act)
    N.call('effdet_bnact_bwd', z, a, nbytes=12.0 * z.numel())          # read dy, z; write dz
    return dz, dgamma, dbeta


def add(a, b):
    out = torch.empty_like(a)
    N.call('effdet_add', a, N.f32(a, 'a'), N.f32(b, 'b'), N.f32(out), a.numel())
    return out


def _contig(t):
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------------------------------------
# Stem   (reference: models/efficientnet.py:193)
# ------------------------------------------------------------------------------------------------


class StemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, gamma, beta, rmean, rvar, eps):
        check_cuda_f32(x, 'EfficientNet input')
        x = _contig(x)
        B, Cin, H, W = x.shape
        if Cin != 3:
            raise N.EffdetNativeError('stem expects 3 input channels, got %d' % Cin)
        C0 = w.shape[0]
        scale, shift, rstd = bn_fold(gamma, beta, rmean, rvar, eps)
        Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
        z = _empty((B, Ho, Wo, C0), x)
        y = _empty((B, Ho, Wo, C0), x)
        wc = _contig(w.detach())
        N.call('effdet_stem_fwd', x, N.f32(x, 'image'), N.f32(wc), N.f32(scale), N.f32(shift), N.f32(z), N.f32(y),
               B, H, W, C0, nbytes=4.0 * (x.numel() + 2 * z.numel()))
        ctx.save_for_backward(x, z, scale, shift, rmean, rstd)
        ctx.C0 = C0
        return y

    @staticmethod
    def backward(ctx, dy):
        x, z, scale, shift, rmean, rstd = ctx.saved_tensors
        dy = _contig(dy)
        B, _, H, W = x.shape
        dz, dgamma, dbeta = bnact_bwd(dy, z, scale, shift, rmean, rstd, ACT_SWISH)
        dw = _zeros((ctx.C0, 3, 3, 3), x)
        N.call('effdet_stem_wgrad', x, N.f32(x), N.f32(dz), N.f32(dw), B, H, W, ctx.C0,
               nbytes=4.0 * (x.numel() + dz.numel()))
        return None, dw, dgamma, dbeta, None, None, None


# ------------------------------------------------------------------------------------------------
# MBConv block   (reference: models/efficientnet.py:75-105)
# ------------------------------------------------------------------------------------------------


class MBConvFn(torch.autograd.Function):
    """args: x (NHWC), row_scale ([B] drop-connect multiplier or None), cfg dict, then parameters
    [We,g0,b0,rm0,rv0]? Wd,g1,b1,rm1,rv1, Wr,br,Wx,bx, Wp,g2,b2,rm2,rv2.

    Only PRE-activations live in HBM, like the reference's MemoryEfficientSwish (models/utils.py:31-42): the expand
    GEMM writes the raw z0, the depthwise kernel applies BN0+swish while staging z0 and writes the raw z1 (its epilogue
    also yields the squeeze-excite mean), the project GEMM applies BN1+swish+gate while staging z1.  Forward = 4
    launches; backward never materialises dz1 / da0 (effdet_dwconv_bwd_fused)."""

    @staticmethod
    def forward(ctx, x, row_scale, cfg, *P):
        x = _contig(x)
        B, H, W, Cin = x.shape
        k, s, eps = cfg['k'], cfg['s'], cfg['eps']
        i = 0
        saved = {}
        if cfg['expand']:
            We, g0, b0, rm0, rv0 = P[0:5]
            i = 5
            sc0, sh0, rs0 = bn_fold(g0, b0, rm0, rv0, eps)
            wf, _ = pack_conv(We)
            z0 = conv2d(x, wf, We.shape[0], 1, w_tc=tc_packs(We)[0])          # raw: BN0 + swish happen in the consumer
            saved.update(z0=z0, sc0=sc0, sh0=sh0, rs0=rs0, rm0=rm0)
            dw_in, isc, ish = z0, sc0, sh0
        else:
            dw_in, isc, ish = x, None, None
        Wd, g1, b1, rm1, rv1, Wr, br, Wx, bx, Wp, g2, b2, rm2, rv2 = P[i:i + 14]
        C = Wd.shape[0]
        sc1, sh1, rs1 = bn_fold(g1, b1, rm1, rv1, eps)
        pt, pl = cfg['pad_t'], cfg['pad_l']
        Ho = (H + cfg['pad_h'] - k) // s + 1
        Wo = (W + cfg['pad_w'] - k) // s + 1
        z1 = _empty((B, Ho, Wo, C), x)
        mean = _zeros((B, C), x)
        wkkc = pack_dw(Wd)
        fa = N.DwFwdArgs(N.f32(dw_in), N.f32(isc), N.f32(ish), N.f32(wkkc), N.f32(sc1), N.f32(sh1), N.f32(z1),
                         N.f32(mean), B, H, W, C, k, s, pt, pl, Ho, Wo, 1.0 / (Ho * Wo))
        N.call('effdet_dwconv_fwd_fused', x, fa, nbytes=4.0 * (dw_in.numel() + z1.numel()))
        # squeeze-excite gate from the mean the depthwise epilogue accumulated
        S = Wr.shape[0]
        s_pre = _empty((B, S), x)
        gate = _empty((B, C), x)
        wr, wx = _contig(Wr.detach()), _contig(Wx.detach())
        N.call('effdet_se_gate_fwd', x, N.f32(mean), N.f32(wr), N.f32(br.detach()), N.f32(wx), N.f32(bx.detach()),
               N.f32(s_pre), N.f32(gate), B, C, S)
        # project: operand swish(bn1(z1)) * gate built while staging, then BN2, drop-connect, skip
        sc2, sh2, rs2 = bn_fold(g2, b2, rm2, rv2, eps)
        wpf, _ = pack_conv(Wp)
        Cout = Wp.shape[0]
        skip = cfg['skip']
        y, z2 = conv2d(z1, wpf, Cout, 1, scale=sc2, shift=sh2, a_scale=gate, in_scale=sc1, in_shift=sh1,
                       row_scale=row_scale if skip else None, residual=x if skip else None, save_z=True,
                       w_tc=tc_packs(Wp)[0])
        ctx.cfg = cfg
        ctx.P = P
        ctx.t = dict(saved, x=x, z1=z1, mean=mean, s_pre=s_pre, gate=gate, z2=z2, sc1=sc1, sh1=sh1,
                     rs1=rs1, rm1=rm1, sc2=sc2, sh2=sh2, rs2=rs2, rm2=rm2, row_scale=row_scale if skip else None,
                     wkkc=wkkc, dims=(B, H, W, Ho, Wo))
        return y

    @staticmethod
    def backward(ctx, dy):
        cfg, P, t = ctx.cfg, ctx.P, _stash(ctx, 't')
        if t is None:
            raise RuntimeError('MBConvFn: backward called twice (activations are released after the first backward)')
        dy = _contig(dy)
        x = t['x']
        B, H, W, Ho, Wo = t['dims']
        k, s = cfg['k'], cfg['s']
        expand = cfg['expand']
        i = 5 if expand else 0
        Wd, g1, b1, rm1, rv1, Wr, br, Wx, bx, Wp, g2, b2, rm2, rv2 = P[i:i + 14]
        C = Wd.shape[0]
        z1, gate = t['z1'], t['gate']
        # project BN (no activation), drop-connect scale folded in
        dz2, dg2, db2 = bnact_bwd(dy, t['z2'], t['sc2'], t['sh2'], t['rm2'], t['rs2'], ACT_NONE,
                                  row_scale=t['row_scale'])
        zb = _zeros_like_many([Wp, Wr, br, Wx, bx, Wd, g1, b1] + ([P[0], P[1], P[2]] if expand else []))
        dWp = zb[0]
        conv_wgrad(z1, dz2, dWp, None, 1, a_scale=gate, tc=tc_enabled(), in_scale=t['sc1'], in_shift=t['sh1'])
        _, wpd = pack_conv(Wp)
        dq = conv2d(dz2, wpd, C, 1, w_tc=tc_packs(Wp)[1])     # grad w.r.t. (a1 * gate)
        # squeeze-excite backward: dgate = sum_px dq * swish(bn1(z1)) with the activation recomputed
        dgate = _zeros((B, C), x)
        N.call('effdet_spatial_reduce_act', x, N.f32(dq), N.f32(z1), N.f32(t['sc1']), N.f32(t['sh1']), N.f32(dgate), 1.0,
               B, Ho * Wo, C, nbytes=8.0 * z1.numel())
        S = Wr.shape[0]
        dmean = _empty((B, C), x)
        dWr, dbr, dWx, dbx = zb[1], zb[2], zb[3], zb[4]
        se_ws = _empty((B * (C + S),), x)
        N.call('effdet_se_gate_bwd', x, N.f32(dgate), N.f32(t['mean']), N.f32(t['s_pre']), N.f32(gate),
               N.f32(_contig(Wr.detach())), N.f32(_contig(Wx.detach())), N.f32(dmean), N.f32(dWr), N.f32(dbr),
               N.f32(dWx), N.f32(dbx), N.f32(se_ws), B, C, S)
        # BN1+swish backward (SE product rule), depthwise weight + data gradient, BN0+swish backward: one pass
        dWd, dg1, db1 = zb[5], zb[6], zb[7]
        dw_in = t['z0'] if expand else x
        dg0 = db0 = None
        if expand:
            dg0, db0 = zb[9], zb[10]
        # with an expand conv the gradient of its raw output is consumed only by tensor-core GEMMs (data + weight
        # gradient): the kernel writes it as bf16 hi/lo planes, the operand format, instead of fp32 + a split pass
        planes = split_planes_like(dw_in) if expand and planes_ok(B, H, W, C) else None
        dxe = None if planes is not None else _empty((B, H, W, C), x)
        ba = N.DwBwdArgs(N.f32(dq), N.f32(z1), N.f32(gate), N.f32(dmean), N.f32(t['sc1']), N.f32(t['sh1']),
                         N.f32(t['rm1'], 'mean'), N.f32(t['rs1']), N.f32(dw_in),
                         N.f32(t['sc0']) if expand else None, N.f32(t['sh0']) if expand else None,
                         N.f32(t['rm0'], 'mean') if expand else None, N.f32(t['rs0']) if expand else None,
                         N.f32(t['wkkc']), N.f32(dxe), N.f32(dWd), N.f32(dg1), N.f32(db1), N.f32(dg0), N.f32(db0),
                         1.0 / (Ho * Wo), B, H, W, C, k, s, cfg['pad_t'], cfg['pad_l'], Ho, Wo,
                         N.ptr(planes))
        N.call('effdet_dwconv_bwd_fused', x, ba, nbytes=4.0 * (2 * z1.numel() + 2 * dw_in.numel()))
        grads = []
        if expand:
            We = P[0]
            dWe = zb[8]
            _, wed = pack_conv(We)
            if planes is not None:
                conv_wgrad_raw(x, N.f32(x, 'x'), H * W * x.shape[3], None, H * W * C, dWe, None, B, H, W, x.shape[3], C, 1,
                               tc=True, dy_planes=planes)
                dx = conv2d_from_planes(planes, wed, x.shape[3], residual=dy if cfg['skip'] else None, w_tc=tc_packs(We)[1])
            else:
                conv_wgrad(x, dxe, dWe, None, 1, tc=tc_enabled())
                dx = conv2d(dxe, wed, x.shape[3], 1, residual=dy if cfg['skip'] else None, w_tc=tc_packs(We)[1])
            grads += [dWe, dg0, db0, None, None]
        else:
            dx = add(dxe, dy) if cfg['skip'] else dxe
        grads += [dWd, dg1, db1, None, None, dWr, dbr, dWx, dbx, dWp, dg2, db2, None, None]
        ctx.t = None
        return (dx, None, None) + tuple(grads)


# ------------------------------------------------------------------------------------------------
# Generic ConvModule: conv + bias (+ReLU)   (reference: models/module.py:507-515)
# ------------------------------------------------------------------------------------------------


class ConvBiasActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act):
        x = _contig(x)
        k = w.shape[2]
        wf, _ = pack_conv(w)
        y = conv2d(x, wf, w.shape[0], k, bias=b.detach() if b is not None else None, act=act, w_tc=tc_packs(w)[0])
        ctx.save_for_backward(x, y if act == ACT_RELU else None)
        ctx.w, ctx.b, ctx.act = w, b, act
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        w, b = ctx.w, ctx.b
        dy = _contig(dy)
        if ctx.act == ACT_RELU:
            dz = torch.empty_like(dy)
            N.call('effdet_relu_bwd', dy, N.f32(dy), N.f32(y), N.f32(dz), dy.numel())
        else:
            dz = dy
        k = w.shape[2]
        dw = torch.zeros_like(w)
        db = torch.zeros_like(b) if b is not None else None
        conv_wgrad(x, dz, dw, db, k, tc=tc_enabled())
        dx = None
        if ctx.needs_input_grad[0]:
            _, wd = pack_conv(w)
            dx = conv2d(dz, wd, x.shape[3], k, w_tc=tc_packs(w)[1])
        return dx, dw, db, None


# ------------------------------------------------------------------------------------------------
# One BiFPN layer   (reference: BiFPNModule.forward, models/bifpn.py:172-203)
# ------------------------------------------------------------------------------------------------


def _fuse_fwd(a, b, c, w, col, eps, mode, planes=False):
    B, H, W, C = a.shape
    # the reference fails with a shape mismatch in `w*in + w*F.interpolate(...)` (models/bifpn.py:188-201) when the
    # pyramid does not halve exactly; the kernels index b as [y//2, x//2] / [2y+dy, 2x+dx], so refuse the same inputs
    want = (B, H // 2, W // 2, C) if mode == FUSE_UP else (B, 2 * H, 2 * W, C)
    if tuple(b.shape) != want or (mode == FUSE_UP and (H % 2 or W % 2)) or (c is not None and c.shape != a.shape):
        raise N.EffdetNativeError('BiFPN levels must halve exactly (image height and width multiples of 128): node '
                                  'input %s cannot be fused with %s' % (tuple(a.shape), tuple(b.shape)))
    out = _planes(B, H, W, C, a) if planes else torch.empty_like(a)      # planes: the node conv's TMA operand format
    wst = w.shape[1]
    args = N.FuseArgs(N.f32(a), N.f32(b), N.f32(c), w.data_ptr() + 4 * col, wst, eps, None if planes else N.f32(out),
                      B, H, W, C, mode, N.ptr(out) if planes else None)
    N.call('effdet_bifpn_fuse_fwd', a, args,
           nbytes=4.0 * (2 * a.numel() + b.numel() + (c.numel() if c is not None else 0)))
    return out


def _fuse_bwd(dout, a, b, c, w, col, eps, mode, da, acc_a, db, acc_b, dc, acc_c, dw):
    B, H, W, C = a.shape
    scratch = _zeros((4,), a)
    wst = w.shape[1]
    args = N.FuseBwdArgs(N.f32(dout), N.f32(a), N.f32(b), N.f32(c), w.data_ptr() + 4 * col, wst, eps, N.f32(da),
                         N.f32(db), N.f32(dc), acc_a, acc_b, acc_c, dw.data_ptr() + 4 * col, N.f32(scratch),
                         B, H, W, C, mode)
    N.call('effdet_bifpn_fuse_bwd', a, args,
           nbytes=4.0 * (3 * a.numel() + 2 * b.numel() + (2 * c.numel() if c is not None else 0)))


class BiFPNLayerFn(torch.autograd.Function):
    """args: eps, L, in[0..L-1] (NHWC, fine->coarse), w1 [2,L], w2 [3,L-2], then (weight, bias) x 2(L-1)."""

    @staticmethod
    def forward(ctx, eps, L, *args):
        ins = [_contig(t) for t in args[:L]]
        w1, w2 = args[L], args[L + 1]
        convs = args[L + 2:]
        w1c, w2c = _contig(w1.detach()), _contig(w2.detach())
        C = ins[0].shape[3]

        # tensor-core mode: the fused map is written as bf16 hi/lo planes and the node conv is the TMA-fed planes
        # kernel (no gather, no split pass in the weight gradient); every level must admit a TMA pixel box
        pl = tc_enabled() and C % 4 == 0 and pixel_boxes_ok(t.shape for t in ins)

        def conv(idx, f, like):
            if pl:
                B_, H_, W_, _ = like.shape
                y = _empty((B_, H_, W_, C), like)
                conv_planes_multi(like, [dict(x=f, y_ptr=N.f32(y), y_bs=H_ * W_ * C, B=B_, H=H_, W=W_)],
                                  tc_packs(convs[2 * idx])[0], C, C, 3, bias=convs[2 * idx + 1].detach())
                return y
            wf, _ = pack_conv(convs[2 * idx])
            return conv2d(f, wf, C, 3, bias=convs[2 * idx + 1].detach(), w_tc=tc_packs(convs[2 * idx])[0])

        fused = [None] * (2 * (L - 1))
        td = [None] * L
        td[L - 1] = ins[L - 1]
        idx = 0
        for i in range(L - 1, 0, -1):                       # top-down
            f = _fuse_fwd(ins[i - 1], td[i], None, w1c, i - 1, eps, FUSE_UP, planes=pl)
            fused[idx] = f
            td[i - 1] = conv(idx, f, ins[i - 1])
            idx += 1
        out = [None] * L
        out[0] = td[0]
        for i in range(0, L - 2):                           # bottom-up
            f = _fuse_fwd(td[i + 1], out[i], ins[i + 1], w2c, i, eps, FUSE_POOL, planes=pl)
            fused[idx] = f
            out[i + 1] = conv(idx, f, td[i + 1])
            idx += 1
        f = _fuse_fwd(ins[L - 1], out[L - 2], None, w1c, L - 1, eps, FUSE_POOL, planes=pl)   # top level
        fused[idx] = f
        out[L - 1] = conv(idx, f, ins[L - 1])
        ctx.eps, ctx.L, ctx.pl = eps, L, pl
        ctx.keep = (ins, td, out, fused, w1, w2, w1c, w2c, convs)
        return tuple(out)

    @staticmethod
    def backward(ctx, *douts):
        eps, L = ctx.eps, ctx.L
        ins, td, out, fused, w1, w2, w1c, w2c, convs = _stash(ctx, 'keep')
        douts = [_contig(d) for d in douts]
        C = ins[0].shape[3]
        zb = _zeros_like_many([w1c, w2c] + list(convs))
        dw1, dw2 = zb[0], zb[1]
        dconv = [None] * len(convs)

        def conv_bwd(idx, dy):
            w, b = convs[2 * idx], convs[2 * idx + 1]
            dw, db = zb[2 + 2 * idx], zb[3 + 2 * idx]
            dconv[2 * idx], dconv[2 * idx + 1] = dw, db
            if ctx.pl:
                B_, H_, W_, _ = dy.shape
                dyp = _planes(B_, H_, W_, C, dy)           # one pass: planes of dy + the bias gradient (column sums)
                to_planes(N.f32(dy), H_ * W_ * C, dyp, B_, H_ * W_, C, dy, colsum=db)
                wgrad_planes_multi(dy, [dict(x=fused[idx], dy=dyp, B=B_, H=H_, W=W_)], dw, C, C, 3)
                df = _empty((B_, H_, W_, C), dy)
                conv_planes_multi(dy, [dict(x=dyp, y_ptr=N.f32(df), y_bs=H_ * W_ * C, B=B_, H=H_, W=W_)], tc_packs(w)[1], C, C, 3)
                return df
            conv_wgrad(fused[idx], dy, dw, db, 3, tc=tc_enabled())
            _, wd = pack_conv(w)
            return conv2d(dy, wd, C, 3, w_tc=tc_packs(w)[1])

        g_in = [None] * L
        g_td = [None] * L
        g_out = [None] * L
        # top level: out[L-1] = conv_last(fuse_pool(in[L-1], out[L-2]))
        idx = 2 * (L - 1) - 1
        df = conv_bwd(idx, douts[L - 1])
        g_in[L - 1] = torch.empty_like(ins[L - 1])
        buf = torch.empty_like(out[L - 2])
        _fuse_bwd(df, ins[L - 1], out[L - 2], None, w1c, L - 1, eps, FUSE_POOL, g_in[L - 1], 0, buf, 0, None, 0, dw1)
        g_out[L - 2] = add(douts[L - 2], buf)
        # bottom-up nodes in reverse
        for i in range(L - 3, -1, -1):
            idx -= 1
            df = conv_bwd(idx, g_out[i + 1])
            g_td[i + 1] = torch.empty_like(td[i + 1])
            g_in[i + 1] = torch.empty_like(ins[i + 1])
            buf = torch.empty_like(out[i])
            _fuse_bwd(df, td[i + 1], out[i], ins[i + 1], w2c, i, eps, FUSE_POOL, g_td[i + 1], 0, buf, 0,
                      g_in[i + 1], 0, dw2)
            g = add(douts[i], buf)
            if i == 0:
                g_td[0] = g                                  # out[0] is td[0]
            else:
                g_out[i] = g
        # top-down nodes in reverse of their forward order
        for i in range(1, L):
            idx = L - 1 - i
            df = conv_bwd(idx, g_td[i - 1])
            if i - 1 == 0:
                g_in[0] = torch.empty_like(ins[0])
                acc_a = 0
            else:
                acc_a = 1
            db_t = g_in[L - 1] if i == L - 1 else g_td[i]
            _fuse_bwd(df, ins[i - 1], td[i], None, w1c, i - 1, eps, FUSE_UP, g_in[i - 1], acc_a, db_t, 1, None, 0, dw1)
        ctx.keep = None
        return (None, None) + tuple(g_in) + (dw1, dw2) + tuple(dconv)


# ------------------------------------------------------------------------------------------------
# RetinaHead over all pyramid levels   (reference: models/retinahead.py:109-132)
# ------------------------------------------------------------------------------------------------


class RetinaHeadFn(torch.autograd.Function):
    """args: nlevels, num_anchors, num_classes, stacked, feats..., then parameters in the order
    cls_convs (w,b)*stacked, reg_convs (w,b)*stacked, retina_cls w,b, retina_reg w,b.
    Returns (cls [B, sum(HWA), K] after sigmoid, reg [B, sum(HWA), 4]) -- already concatenated.
    Every layer runs on all pyramid levels in one launch (the weights are shared between levels)."""

    @staticmethod
    def forward(ctx, nl, A, K, stacked, *args):
        feats = [_contig(t) for t in args[:nl]]
        P = args[nl:]
        cls_p, reg_p = P[:2 * stacked], P[2 * stacked:4 * stacked]
        wc, bc, wr, br = P[4 * stacked:4 * stacked + 4]
        B = feats[0].shape[0]
        F = cls_p[0].shape[0]
        offs, tot = [], 0
        for f in feats:
            offs.append(tot)
            tot += f.shape[1] * f.shape[2] * A
        cls_all = _empty((B, tot, K), feats[0])
        reg_all = _empty((B, tot, 4), feats[0])
        towers = []
        for tp in (cls_p, reg_p):
            acts = [feats]
            cur = feats
            for i in range(stacked):
                wf, _ = pack_conv(tp[2 * i])
                cur = conv2d_multi(cur, wf, F, 3, bias=tp[2 * i + 1].detach(), act=ACT_RELU, w_tc=tc_packs(tp[2 * i])[0])
                acts.append(cur)
            towers.append(acts)          # acts[i][lv]: input of conv i (acts[stacked] = tower output)
        for (acts, w, bias, out, width, act) in ((towers[0], wc, bc, cls_all, K, ACT_SIGMOID),
                                                 (towers[1], wr, br, reg_all, 4, ACT_NONE)):
            wf, _ = pack_conv(w)
            levels = []
            for lv, t in enumerate(acts[stacked]):
                _, H, W, _ = t.shape
                levels.append(dict(x_ptr=N.f32(t), x_bs=H * W * F, y_ptr=N.f32(out) + 4 * offs[lv] * width,
                                   y_bs=tot * width, B=B, H=H, W=W))
            conv2d_multi_raw(feats[0], levels, wf, F, A * width, 3, bias=bias.detach(), act=act, w_tc=tc_packs(w)[0])
        ctx.meta = (nl, A, K, stacked, offs, tot)
        ctx.keep = (feats, P, towers, cls_all)
        return cls_all, reg_all

    @staticmethod
    def backward(ctx, dcls, dreg):
        nl, A, K, stacked, offs, tot = ctx.meta
        feats, P, towers, cls_all = _stash(ctx, 'keep')
        cls_p, reg_p = P[:2 * stacked], P[2 * stacked:4 * stacked]
        wc, bc, wr, br = P[4 * stacked:4 * stacked + 4]
        B = feats[0].shape[0]
        F = cls_p[0].shape[0]
        Cin = feats[0].shape[3]
        dcls, dreg = _contig(dcls), _contig(dreg)
        dzc = torch.empty_like(dcls)
        N.call('effdet_sigmoid_bwd', dcls, N.f32(dcls), N.f32(cls_all), N.f32(dzc), dcls.numel(),
               nbytes=12.0 * dcls.numel())
        gP = _zeros_like_many(P)
        g_cls, g_reg = gP[:2 * stacked], gP[2 * stacked:4 * stacked]
        gwc, gbc, gwr, gbr = gP[4 * stacked:4 * stacked + 4]
        tc = tc_enabled()
        dfeat = None
        for (acts, tp, tg, wl, gwl, gbl, dsrc, width) in ((towers[0], cls_p, g_cls, wc, gwc, gbc, dzc, K),
                                                          (towers[1], reg_p, g_reg, wr, gwr, gbr, dreg, 4)):
            Co = A * width
            top = acts[stacked]
            levels = []
            d = []
            wl_levels = []
            for lv, t in enumerate(top):
                _, H, W, _ = t.shape
                dptr = N.f32(dsrc) + 4 * offs[lv] * width
                wl_levels.append(dict(x_ptr=N.f32(t), x_bs=H * W * F, dy_ptr=dptr, dy_bs=tot * width, B=B, H=H, W=W))
                dl = _empty((B, H, W, F), t)
                d.append(dl)
                levels.append(dict(x_ptr=dptr, x_bs=tot * width, y_ptr=N.f32(dl), y_bs=H * W * F, B=B, H=H, W=W,
                                   mask_ptr=N.f32(t), mask_bs=H * W * F))
            conv_wgrad_multi(feats[0], wl_levels, gwl, gbl, F, Co, 3, tc=tc)
            _, wld = pack_conv(wl)
            conv2d_multi_raw(feats[0], levels, wld, Co, F, 3, w_tc=tc_packs(wl)[1])
            for i in range(stacked - 1, -1, -1):
                xin = acts[i]
                ci = xin[0].shape[3]
                conv_wgrad_multi(feats[0], [dict(x_ptr=N.f32(xin[lv]), x_bs=xin[lv].shape[1] * xin[lv].shape[2] * ci,
                                                 dy_ptr=N.f32(d[lv]), dy_bs=d[lv].shape[1] * d[lv].shape[2] * F,
                                                 B=B, H=xin[lv].shape[1], W=xin[lv].shape[2]) for lv in range(nl)],
                                 tg[2 * i], tg[2 * i + 1], ci, F, 3, tc=tc)
                _, wd = pack_conv(tp[2 * i])
                wdt = tc_packs(tp[2 * i])[1]
                if i > 0:
                    d = conv2d_multi(d, wd, F, 3, w_tc=wdt, masks=xin)
                else:
                    d = conv2d_multi(d, wd, Cin, 3, w_tc=wdt, residuals=dfeat)
            dfeat = d
        ctx.keep = None
        return (None, None, None, None) + tuple(dfeat) + tuple(gP)


def _pitch8(c):
    return (c + 7) // 8 * 8


def _planes(B, H, W, C, like):
    return torch.empty((2, B, H, W, _pitch8(C)), device=like.device, dtype=torch.bfloat16)


def _relu_bits(B, H, W, C, like):
    """one bit per channel of a ReLU layer's planes (bit c % 32 of word c // 32: stored value > 0)"""
    return torch.empty((B, H, W, (C + 31) // 32), device=like.device, dtype=torch.int32)


def to_planes(x_ptr, x_bs, planes, B, HW, C, dev_t, prob_ptr=None, p_bs=0, colsum=None):
    N.call('effdet_to_planes', dev_t, x_ptr, x_bs, prob_ptr, p_bs, N.ptr(planes), N.f32(colsum, 'colsum'), B, HW, C,
           nbytes=8.0 * B * HW * C)


def conv_planes_multi(dev_t, levels, w_tc, Cin, Cout, k, bias=None, act=ACT_NONE, colsum=None):
    """One launch over the pyramid levels; levels: dicts with x (planes), B, H, W and y_planes and / or (y_ptr, y_bs),
    optional y_mask (_relu_bits the ReLU forward writes), mask (planes) or mask_bits (a y_mask), res_ptr / res_bs."""
    nl = len(levels)
    arr = (N.ConvPlanesArgs * nl)()
    for i, lv in enumerate(levels):
        arr[i] = N.ConvPlanesArgs(N.ptr(lv['x']), w_tc.data_ptr(), N.f32(bias, 'bias'), lv.get('y_ptr'), lv.get('y_bs', 0),
                                  N.ptr(lv.get('y_planes')), N.ptr(lv.get('mask')), lv.get('res_ptr'), lv.get('res_bs', 0),
                                  N.f32(colsum, 'colsum'), lv['B'], lv['H'], lv['W'], Cin, Cout, k, act, tc_single(k),
                                  N.ptr(lv.get('y_mask')), N.ptr(lv.get('mask_bits')))
    px = sum(lv['B'] * lv['H'] * lv['W'] for lv in levels)
    N.call('effdet_conv_planes_multi', dev_t, arr, nl, flops=2.0 * px * k * k * Cin * Cout,
           nbytes=4.0 * (px * (Cin + Cout) + k * k * Cin * Cout))


def wgrad_planes_multi(dev_t, levels, dw, Cin, Cout, k):
    """weight gradient of one shared-weight layer from operands that already live as planes (no split pass);
    levels: dicts with x (planes), dy (planes), B, H, W."""
    nl = len(levels)
    arr = (N.WgradArgs * nl)()
    ws_dw = _ws_dw(dev_t, Cin, Cout, k)
    for i, lv in enumerate(levels):
        arr[i] = N.WgradArgs(None, 0, None, 0, N.f32(dw, 'dw'), None, None, lv['B'], lv['H'], lv['W'], Cin, Cout, k, 1, None,
                             None, None, None, N.ptr(lv['dy']), N.ptr(lv['x']), tc_single(k),
                             ws_dw.data_ptr() if ws_dw is not None else None)
    N.call('effdet_conv2d_wgrad_multi', dev_t, arr, nl)


def head_planes_ok(feats, params):
    """can the RetinaHead run with activations kept as bf16 hi/lo planes (TMA-fed tensor-core path)?"""
    if not tc_enabled() or any(f.shape[3] % 4 for f in feats) or not pixel_boxes_ok(f.shape for f in feats):
        return False
    return all(p.shape[0] % 4 == 0 and p.shape[0] >= 16 for p in params[0::2])


class RetinaHeadPlanesFn(torch.autograd.Function):
    """RetinaHeadFn with every tower activation (and every tower gradient) stored as bf16 hi/lo planes: each conv is ONE
    TMA-fed tensor-core launch over all levels, data gradients hand the bias gradient of the previous layer over as a
    by-product of their epilogue, weight gradients read both operands as they lie -- no split pass, no fp32 tower
    tensors.  Same arguments / results as RetinaHeadFn (models/retinahead.py:109-132)."""

    @staticmethod
    def forward(ctx, nl, A, K, stacked, *args):
        feats = [_contig(t) for t in args[:nl]]
        P = args[nl:]
        cls_p, reg_p = P[:2 * stacked], P[2 * stacked:4 * stacked]
        wc, bc, wr, br = P[4 * stacked:4 * stacked + 4]
        dev_t = feats[0]
        B = feats[0].shape[0]
        Cin = feats[0].shape[3]
        F = cls_p[0].shape[0]
        geo = [(f.shape[0], f.shape[1], f.shape[2]) for f in feats]
        offs, tot = [], 0
        for f in feats:
            offs.append(tot)
            tot += f.shape[1] * f.shape[2] * A
        cls_all = _empty((B, tot, K), dev_t)
        reg_all = _empty((B, tot, 4), dev_t)
        fp = []
        for f in feats:                                    # the BiFPN features as planes, shared by both towers
            pl = _planes(f.shape[0], f.shape[1], f.shape[2], Cin, f)
            to_planes(N.f32(f), f.shape[1] * f.shape[2] * Cin, pl, f.shape[0], f.shape[1] * f.shape[2], Cin, dev_t)
            fp.append(pl)
        towers, tower_bits = [], []
        for tp in (cls_p, reg_p):
            acts, bits = [fp], [None]                      # bits[i]: the ReLU mask of acts[i], for the data gradient
            cur, ci = fp, Cin
            for i in range(stacked):
                nxt = [_planes(b, h, w, F, dev_t) for (b, h, w) in geo]
                nbits = [_relu_bits(b, h, w, F, dev_t) for (b, h, w) in geo]
                conv_planes_multi(dev_t, [dict(x=cur[l], y_planes=nxt[l], y_mask=nbits[l], B=geo[l][0], H=geo[l][1], W=geo[l][2])
                                          for l in range(nl)],
                                  tc_packs(tp[2 * i])[0], ci, F, 3, bias=tp[2 * i + 1].detach(), act=ACT_RELU)
                acts.append(nxt)
                bits.append(nbits)
                cur, ci = nxt, F
            towers.append(acts)
            tower_bits.append(bits)
        for (acts, w, bias, out, width, act) in ((towers[0], wc, bc, cls_all, K, ACT_SIGMOID),
                                                 (towers[1], wr, br, reg_all, 4, ACT_NONE)):
            levels = [dict(x=acts[stacked][l], y_ptr=N.f32(out) + 4 * offs[l] * width, y_bs=tot * width, B=geo[l][0], H=geo[l][1],
                           W=geo[l][2]) for l in range(nl)]
            conv_planes_multi(dev_t, levels, tc_packs(w)[0], F, A * width, 3, bias=bias.detach(), act=act)
        ctx.meta = (nl, A, K, stacked, offs, tot, geo, Cin, F)
        ctx.keep = (P, towers, tower_bits, cls_all)
        return cls_all, reg_all

    @staticmethod
    def backward(ctx, dcls, dreg):
        nl, A, K, stacked, offs, tot, geo, Cin, F = ctx.meta
        if ctx.keep is None:
            raise RuntimeError('RetinaHeadPlanesFn: backward called twice (activations are released after the first backward)')
        P, towers, tower_bits, cls_all = _stash(ctx, 'keep')
        cls_p, reg_p = P[:2 * stacked], P[2 * stacked:4 * stacked]
        wc, bc, wr, br = P[4 * stacked:4 * stacked + 4]
        dcls, dreg = _contig(dcls), _contig(dreg)
        dev_t = dcls
        gP = _zeros_like_many(P)
        g_cls, g_reg = gP[:2 * stacked], gP[2 * stacked:4 * stacked]
        gwc, gbc, gwr, gbr = gP[4 * stacked:4 * stacked + 4]
        dfeat = None
        for (acts, bits, tp, tg, wl, gwl, gbl, dsrc, prob, width) in (
                (towers[0], tower_bits[0], cls_p, g_cls, wc, gwc, gbc, dcls, cls_all, K),
                (towers[1], tower_bits[1], reg_p, g_reg, wr, gwr, gbr, dreg, None, 4)):
            Co = A * width
            # gradient w.r.t. the head outputs -> planes (sigmoid backward folded in) + bias gradient of the output conv
            d = []
            for l, (b, h, w) in enumerate(geo):
                pl = _planes(b, h, w, Co, dev_t)
                to_planes(N.f32(dsrc) + 4 * offs[l] * width, tot * width, pl, b, h * w, Co, dev_t,
                          prob_ptr=(N.f32(prob) + 4 * offs[l] * width) if prob is not None else None, p_bs=tot * width, colsum=gbl)
                d.append(pl)
            top = acts[stacked]
            wgrad_planes_multi(dev_t, [dict(x=top[l], dy=d[l], B=geo[l][0], H=geo[l][1], W=geo[l][2]) for l in range(nl)],
                               gwl, F, Co, 3)
            nxt = [_planes(b, h, w, F, dev_t) for (b, h, w) in geo]
            conv_planes_multi(dev_t, [dict(x=d[l], y_planes=nxt[l], mask_bits=bits[stacked][l], B=geo[l][0], H=geo[l][1], W=geo[l][2])
                                      for l in range(nl)], tc_packs(wl)[1], Co, F, 3, colsum=tg[2 * (stacked - 1) + 1])
            d = nxt
            for i in range(stacked - 1, -1, -1):
                xin = acts[i]
                ci = Cin if i == 0 else F
                wgrad_planes_multi(dev_t, [dict(x=xin[l], dy=d[l], B=geo[l][0], H=geo[l][1], W=geo[l][2]) for l in range(nl)],
                                   tg[2 * i], ci, F, 3)
                wdt = tc_packs(tp[2 * i])[1]
                if i > 0:
                    nxt = [_planes(b, h, w, F, dev_t) for (b, h, w) in geo]
                    conv_planes_multi(dev_t, [dict(x=d[l], y_planes=nxt[l], mask_bits=bits[i][l], B=geo[l][0], H=geo[l][1], W=geo[l][2])
                                              for l in range(nl)], wdt, F, F, 3, colsum=tg[2 * (i - 1) + 1])
                    d = nxt
                else:
                    out = [_empty((b, h, w, Cin), dev_t) for (b, h, w) in geo]
                    conv_planes_multi(dev_t, [dict(x=d[l], y_ptr=N.f32(out[l]), y_bs=geo[l][1] * geo[l][2] * Cin,
                                                   res_ptr=N.f32(dfeat[l]) if dfeat is not None else None,
                                                   res_bs=geo[l][1] * geo[l][2] * Cin, B=geo[l][0], H=geo[l][1], W=geo[l][2])
                                              for l in range(nl)], wdt, F, Cin, 3)
                    dfeat = out
        ctx.keep = None
        return (None, None, None, None) + tuple(dfeat) + tuple(gP)


# ------------------------------------------------------------------------------------------------
# FocalLoss   (reference: models/losses.py:32-152)
# ------------------------------------------------------------------------------------------------


# Annotation rows per image that effdet_focal_loss_fwd / _bwd stage in shared memory at once; wider tables, and calls
# with device-side counts, go through the counted pair, which stages them in chunks of this many rows.
FOCAL_MAX_G = 256


def annotation_counts(B, G, device):
    """[1 + B] int32 on the device: (B, G, ..., G), every image and every row.  Two fills, no host read."""
    counts = torch.full((1 + B,), G, dtype=torch.int32, device=device)
    counts[:1].fill_(B)
    return counts


class FocalLossFn(torch.autograd.Function):
    """counts: None, or [1 + B] int32 on the device (include/effdet_b200.h, effdet_focal_loss_counted_fwd): counts[0]
    real images (the loss is their mean), counts[1 + b] annotation rows of image b.  With counts, or with more than
    FOCAL_MAX_G annotation rows, the counted entry points run; otherwise the uncounted pair."""

    @staticmethod
    def forward(ctx, cls, reg, anchors, annots, alpha, gamma, counts=None):
        check_cuda_f32(cls, 'classifications')
        check_cuda_f32(reg, 'regressions')
        cls, reg = _contig(cls), _contig(reg)
        anchors = _contig(anchors.to(device=cls.device, dtype=torch.float32))
        annots = _contig(annots.to(device=cls.device, dtype=torch.float32))
        B, A, K = cls.shape
        G = annots.shape[1]
        if (counts is not None or G > FOCAL_MAX_G) and tuple(annots.shape) != (B, G, 5):
            raise N.EffdetNativeError('FocalLoss: annotations must be [B=%d, G, 5], got %s' % (B, tuple(annots.shape)))
        if counts is not None:
            if counts.dtype != torch.int32 or counts.numel() != 1 + B or counts.device != cls.device:
                raise N.EffdetNativeError('FocalLoss: counts must be a [1 + B] = [%d] int32 tensor on %s, got %s %s on %s'
                                          % (1 + B, cls.device, tuple(counts.shape), counts.dtype, counts.device))
            counts = _contig(counts)
        elif G > FOCAL_MAX_G:
            counts = annotation_counts(B, G, cls.device)
        losses = _empty((2,), cls)
        assign = torch.empty((B, A), device=cls.device, dtype=torch.int32)
        stats = _empty((B, 4), cls)
        if counts is None:
            N.call('effdet_focal_loss_fwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4)), N.f32(annots),
                   N.f32(losses), assign.data_ptr(), N.f32(stats), B, A, K, G, float(alpha), float(gamma),
                   nbytes=4.0 * (cls.numel() + reg.numel()))
            ctx.save_for_backward(cls, reg, anchors, annots, assign, stats)
        else:
            N.call('effdet_focal_loss_counted_fwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4)),
                   N.f32(annots), N.ptr(counts), N.f32(losses), assign.data_ptr(), N.f32(stats), B, A, K, G, float(alpha),
                   float(gamma), nbytes=4.0 * (cls.numel() + reg.numel()))
            ctx.save_for_backward(cls, reg, anchors, annots, assign, stats, counts)
        ctx.hp = (float(alpha), float(gamma))
        return losses.narrow(0, 0, 1), losses.narrow(0, 1, 1)

    @staticmethod
    def backward(ctx, g_cls, g_reg):
        cls, reg, anchors, annots, assign, stats, *counts = ctx.saved_tensors
        B, A, K = cls.shape
        G = annots.shape[1]
        gout = _zeros((2,), cls)
        if g_cls is not None:
            gout[0:1].copy_(g_cls.reshape(1))
        if g_reg is not None:
            gout[1:2].copy_(g_reg.reshape(1))
        dcls, dreg = torch.empty_like(cls), torch.empty_like(reg)
        if not counts:
            N.call('effdet_focal_loss_bwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4)), N.f32(annots),
                   N.f32(gout), assign.data_ptr(), N.f32(stats), N.f32(dcls), N.f32(dreg), B, A, K, G, ctx.hp[0],
                   ctx.hp[1], nbytes=8.0 * (cls.numel() + reg.numel()))
        else:
            N.call('effdet_focal_loss_counted_bwd', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4)),
                   N.f32(annots), N.ptr(counts[0]), N.f32(gout), assign.data_ptr(), N.f32(stats), N.f32(dcls),
                   N.f32(dreg), B, A, K, G, ctx.hp[0], ctx.hp[1], nbytes=8.0 * (cls.numel() + reg.numel()))
        return dcls, dreg, None, None, None, None, None


def pack_annotations(annots, out, counts):
    """Copy a ragged collated batch annots [B, G, 5] (-1 padded, B <= Bcap, G <= Gcap) into the static table out
    [Bcap, Gcap, 5] and counts [1 + Bcap] (effdet_pack_annots): each image's labelled rows first, in order.  One launch,
    no host read."""
    B, G = annots.shape[0], annots.shape[1]
    N.call('effdet_pack_annots', out, N.f32(annots), B, G, N.f32(out), N.ptr(counts), out.shape[0], out.shape[1])


# ------------------------------------------------------------------------------------------------
# Inference post-processing   (reference: models/efficientdet.py:70-86)
# ------------------------------------------------------------------------------------------------


# Bytes the NMS workspace may take before the batch is split into consecutive groups of images (at least one image per
# group).  Realistic candidate counts keep the whole batch in one group: 5 k candidates cost 3.2 MB per image.
NMS_MASK_BUDGET = 1 << 30

# Column chunk of the NMS for cap > NMS_CHUNK (effdet_nms_batch_chunked): the workspace is NMS_CHUNK * NMS_CHUNK / 8
# bytes of mask per image (2 MiB at 4096), whatever the candidate count.  Up to NMS_CHUNK candidates NMS runs as one
# chunk, which is the square-mask path.  4096 keeps every realistic candidate count (a few thousand) on that path
# unchanged.  Measured (tools/bench_detect.py chunk_sweep; H100 80GB HBM3, 700 W), chunk 1024 / 2048 / 4096 / 8192:
# D0 512^2 bs 32 with all 49 104 anchors 16.4 / 16.4 / 17.9 / 22.3 ms, the D7 bench image (327 867 candidates)
# 52.5 / 49.7 / 49.5 / 49.3 ms.
NMS_CHUNK = 4096

Detections = collections.namedtuple('Detections', 'scores classes boxes count')


def candidate_cap(max_candidates, cls):
    """the fixed cap detect_batch gets for cls [B,A,K]: max_candidates clamped to A, or A for None"""
    A = cls.shape[1]
    return A if max_candidates is None else min(int(max_candidates), A)


def _nms_workspace(B, cap, chunk):
    """bytes of effdet_nms_batch_chunked's workspace"""
    n = int(N.load().effdet_nms_chunked_workspace(B, cap, chunk))
    if n < 0:
        raise N.EffdetNativeError('detect_batch: %s' % N.last_error())
    return n


def detect_batch(cls, reg, anchors, img_h, img_w, threshold, iou_threshold, cap=None):
    """Decode + clip + class max + threshold + greedy NMS of every image of cls [B,A,K] / reg [B,A,4], one set of
    launches for the whole batch (the reference does this for image 0 only, models/efficientdet.py:73-86).

    cap=None: reads the B candidate counts once to set cap = their maximum and the B kept counts once to slice the
    results -> list of B triples [scores[K_b], classes[K_b] int64, boxes[K_b,4]] on the device (empty tensors when no
    anchor passes the threshold).
    cap=C: no host synchronisation, so the call can be captured in a CUDA graph -> Detections(scores [B,C],
    classes [B,C] int64, boxes [B,C,4], count [B] int32), rows past count[b] zero; count[b] == -1 when image b has
    more than C candidates (its rows are then all zero)."""
    check_cuda_f32(cls, 'classifications')
    check_cuda_f32(reg, 'regressions')
    cls, reg = _contig(cls), _contig(reg)
    B, A, K = cls.shape
    anchors = _contig(anchors.view(-1, 4))
    npad = 1 << (A - 1).bit_length()
    dev = cls.device
    boxes = _empty((B, A, 4), cls)
    scores = _empty((B, A), cls)
    classes = torch.empty((B, A), device=dev, dtype=torch.int32)
    keys = torch.empty((B, npad), device=dev, dtype=torch.int64)
    count = torch.empty((B,), device=dev, dtype=torch.int32)
    N.call('effdet_detect_candidates_batch', cls, N.f32(cls), N.f32(reg), N.f32(anchors), N.f32(boxes), N.f32(scores),
           classes.data_ptr(), keys.data_ptr(), count.data_ptr(), B, A, K, npad, float(img_w), float(img_h),
           float(threshold))
    eager = cap is None
    if eager:
        cap = int(count.max().item())                # host read 1 of 2: sizes the NMS workspace and the outputs
        if cap == 0:
            return [[cls.new_zeros(0), torch.zeros(0, dtype=torch.int64, device=dev), cls.new_zeros(0, 4)]
                    for _ in range(B)]
    chunk = min(cap, NMS_CHUNK)
    per_image = _nms_workspace(1, cap, chunk)
    group = min(B, max(NMS_MASK_BUDGET, per_image) // per_image)
    ws_bytes = _nms_workspace(group, cap, chunk)
    ws = torch.empty((ws_bytes // 8,), device=dev, dtype=torch.int64)
    keep = torch.empty((B, cap), device=dev, dtype=torch.int32)
    nkeep = torch.empty((B,), device=dev, dtype=torch.int32)
    for b0 in range(0, B, group):
        N.call('effdet_nms_batch_chunked', cls, N.f32(boxes[b0:]), keys[b0:].data_ptr(), count[b0:].data_ptr(),
               min(group, B - b0), A, npad, cap, chunk, float(iou_threshold), ws.data_ptr(), ws_bytes,
               keep[b0:].data_ptr(), nkeep[b0:].data_ptr())
    o_s = _empty((B, cap), cls)
    o_c = torch.empty((B, cap), device=dev, dtype=torch.int64)
    o_b = _empty((B, cap, 4), cls)
    N.call('effdet_gather_detections_batch', cls, N.f32(boxes), N.f32(scores), classes.data_ptr(), keep.data_ptr(),
           nkeep.data_ptr(), B, A, cap, N.f32(o_s), o_c.data_ptr(), N.f32(o_b))
    if not eager:
        return Detections(o_s, o_c, o_b, nkeep)
    m = nkeep.tolist()                               # host read 2 of 2
    return [[o_s[b, :m[b]], o_c[b, :m[b]], o_b[b, :m[b]]] for b in range(B)]
