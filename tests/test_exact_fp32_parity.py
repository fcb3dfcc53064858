"""Kernel-level fp64 parity of the exact-fp32 convolutions (EFFDET_B200_PRECISION=fp32) at the calls that mode makes.

In fp32 mode tc_packs() returns no tensor-core packs, so every dense convolution of the network runs on conv_simt.cu:

  conv_igemm_kernel<128,8>, <64,4>, <32,4>   every forward and data gradient, with the prologue (BN1 + swish while the
                                              operand is staged, the squeeze-excite gate) and the epilogue (bias, z,
                                              BN affine, activation, drop-connect row_scale, residual, ReLU mask)
  conv_wgrad_kernel<BC,BN,TC,TN>              every weight gradient, one launch per pyramid level, fp32 atomics
  colsum_kernel                               every bias gradient

This file

  * records the conv calls of one fp32-mode step of bench.CONFIGS d0 and d4 (train) and of the d7 backbone + BiFPN +
    head forward, through the product's host code with the C ABI replaced by tests/test_host_trace.py's Recorder,
    and checks that every level takes the exact-fp32 route (no w_tc, precision 0);
  * mirrors conv_simt_launch, wgrad_simt_launch and colsum_launch in Python (_igemm_plan, _wgrad_plan, _colsum_plan) and
    sorts every recorded level into a plan class; the GPU cases (CASES) must reach every class of the three traces, the
    longest weight-gradient accumulation (32 768 pixels per CTA), the longest reduction (405 K-steps) and the largest
    igemm grid;
  * runs each GPU case once under torch.profiler (kernel names with template arguments, grids), then holds it to a
    float64 reference computed on the device from the same fp32 operands.

Per-element bound (the check with teeth).  The kernels accumulate with fmaf: one rounding per multiply-add, each
|fl(a*b + s) - (a*b + s)| <= u |a*b + s|, u = 2^-24.  A sum of n products formed by any sequence of such operations
(recursive, pairwise, merged by atomics, starting from a non-zero value, which counts as one more term) satisfies
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 3.1 and 4.2)

    |fl(sum) - sum| <= gamma_n * sum |a_i b_i|,    gamma_n = n u / (1 - n u),

with n the longest chain of roundings any term passes through.  So

    |got - ref| <= gamma_n * (|A| (*) |W|) + E_A (*) |W| + e_epi

  |A| (*) |W|   the fp64 convolution (or weight-gradient product) of the absolute operands (plus |dw0| for the initial
                value of a weight gradient);
  n             igemm: taps * Cin (zero-padded channels and taps add exact zeros);
                wgrad: pixels per CTA + splits * levels + 1 (the atomics of every split of every level, and dw0);
                colsum: rows per block + rows of the shared reduction + blocks * levels + 1;
  E_A           the prologue operand's own error, per element: a = swish(x s + t) g is formed in fp32 as
                fl(fl(swish(fl(x s + t))) g).  fmaf rounds x s + t once, which moves swish by at most
                |v swish'(v)| u; expf is within 2 ulp (CUDA C Programming Guide, sec. 'Mathematical Functions'),
                1 + e, the IEEE division, v * sigma and * g round once each:
                |fl(a) - a| <= (|v swish'(v)| + 8 |swish(v)|) |g| u (to first order; every bound is taken with a
                factor 1 + 1e-3 for the second-order terms);
  e_epi         the accumulator's bound carried through the epilogue in the kernel's order with each op's Lipschitz
                constant, plus the op's own rounding of the fp64 value: bias add u|v|; affine fmaf |scale| E + u|v|;
                ReLU E; sigmoid E/4 + 6u sigma (expf 4u, add, division); swish 1.1 E + 7u |swish|;
                row_scale |r| E + u|v|; residual E + u|v|; the ReLU mask keeps or zeroes E.

A correct kernel cannot exceed this bound in any summation order; a wrong tap, tile, row, stride, mask or epilogue order
breaks it element-wise even in a 10^8-element tensor, where a norm would dilute the error.  Every case prints the worst
per-element ratio |got - ref| / bound, which must stay below 1.

Norm-relative bounds (the house style, ||got - ref|| / ||ref||):
  TOL_EXACT = 5e-5  each whole tensor (as tests/test_gpu_parity.py and tests/test_conv_routing.py), each dbias
  TOL_LOCAL = 1e-4  each image, each block of 64 output channels, and each tap of a weight gradient

Negative controls, one per kernel: the igemm reference without one 16-channel K-slice of one tap breaks the
per-element bound on most outputs that slice reaches; the weight-gradient reference without the last 16-pixel chunk of
each split of the first level exceeds TOL_LOCAL on some tap (one chunk alone does not at 2^19 pixels: 3e-5 of a sum
with a mean); the bias-gradient reference without one row block of colsum_kernel exceeds its
per-element bound."""
import collections
import json
import math
import os
import pathlib
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O
from test_benchmark_plans import _launches
from test_host_trace import Recorder

TOL_EXACT = 5e-5
TOL_LOCAL = 1e-4
U = 2.0 ** -24
SMS = 132                       # H100 SXM: the SM count the benchmark's plans are walked at
GUARD = 4096                    # NaN elements after every output buffer
A = 9                           # anchors per pixel
KBM, KBK, KNT = 128, 16, 256    # conv_simt.cu: output pixels per igemm CTA, reduction slice, threads per CTA
ACTS = {0: 'none', 1: 'relu', 2: 'swish', 3: 'sigmoid'}


def _cdiv(a, b):
    return -(-a // b)


def _gamma(n):
    return n * U / (1 - n * U)


# ------------------------------------------------------------------------------------------------
# mirrors of conv_simt_launch, wgrad_simt_launch and colsum_launch (conv_simt.cu, common.cuh)
# ------------------------------------------------------------------------------------------------

def _igemm_plan(B, H, W, Cin, Cout, k):
    """conv_simt_launch: the N tile that pads Cout least (ties to the wider tile), its kernel, K-steps, grid"""
    best, pad = 128, _cdiv(Cout, 128) * 128
    for bn in (64, 32):
        if _cdiv(Cout, bn) * bn < pad:
            best, pad = bn, _cdiv(Cout, bn) * bn
    M = B * H * W
    return dict(BN=best, kernel='conv_igemm_kernel<%d,%d>(' % (best, 8 if best == 128 else 4),
                ksteps=k * k * _cdiv(Cin, KBK), grid=(_cdiv(M, KBM), _cdiv(Cout, best), 1),
                partial_m=M % KBM != 0, tail=Cout % best)


def _wgrad_plan(B, H, W, Cin, Cout, k, sms=SMS):
    """wgrad_simt_launch: instantiation, tiles, splits of about three waves (each at least 16 chunks), chunks per
    split, pixels one CTA accumulates, grid"""
    if Cin <= 32:
        inst = (32, 128, 4, 4)
    elif Cout <= 48:
        inst = (128, 32, 4, 4)
    elif Cin >= 128 and Cout >= 128:
        inst = (128, 128, 8, 8)
    else:
        inst = (64, 64, 4, 4)
    ctiles, ntiles = _cdiv(Cin, inst[0]), _cdiv(Cout, inst[1])
    nchunks = _cdiv(B * H * W, KBK)
    splits = max(1, _cdiv(sms * 3, ctiles * ntiles * k * k))
    splits = min(splits, _cdiv(nchunks, 16))
    cps = _cdiv(nchunks, splits)
    splits = _cdiv(nchunks, cps)
    return dict(inst=inst, kernel='conv_wgrad_kernel<%d,%d,%d,%d>(' % inst, ctiles=ctiles, ntiles=ntiles,
                nchunks=nchunks, cps=cps, splits=splits, pixels=cps * KBK, grid=(ctiles * ntiles, k * k, splits))


def _colsum_plan(M, N, sms=SMS):
    """colsum_launch: rows of the shared reduction (rowpack_rows), rows per block (about four waves, at least 8 row
    iterations), grid"""
    cvecs = N // 4
    rows = 1 if cvecs >= KNT else KNT // cvecs
    rpb = max(_cdiv(M, sms * 4), rows * 8)
    return dict(rows=rows, rpb=rpb, grid=(_cdiv(M, rpb), 1 if cvecs <= KNT else _cdiv(cvecs, KNT), 1))


# ------------------------------------------------------------------------------------------------
# plan classes of one conv level / one weight-gradient level
# ------------------------------------------------------------------------------------------------

PROLOGUE = ('in_scale', 'a_scale')
EPILOGUE = ('bias', 'z', 'scale', 'row_scale', 'residual', 'mask_src')


def _classes(kind, levels):
    """-> [(plan class, figure)] of one recorded call: for a conv level (igemm, BN tile, ksize, prologue, epilogue,
    strided x, strided y, partial last M tile, Cout tail) with its grid size; for a weight-gradient level (wgrad,
    instantiation, ksize, prologue, strided dy, multi-level) with its pixels per CTA, and (colsum, rows of the shared
    reduction) with its rows per block"""
    out = []
    for a in levels:
        B, H, W, Cin, Cout, k = (a[f] for f in ('B', 'H', 'W', 'Cin', 'Cout', 'ksize'))
        pro = tuple(f for f in PROLOGUE if a[f] is not None)
        if kind != 'wgrad':
            p = _igemm_plan(B, H, W, Cin, Cout, k)
            epi = tuple(f for f in EPILOGUE if a[f] is not None) + (ACTS[a['act']],)
            out.append((('igemm', p['BN'], k, pro, epi, a['x_bstride'] != H * W * Cin, a['y_bstride'] != H * W * Cout,
                         p['partial_m'], p['tail'] != 0), p['grid'][0] * p['grid'][1]))
        else:
            p = _wgrad_plan(B, H, W, Cin, Cout, k)
            out.append((('wgrad', p['inst'], k, pro, a['dy_bstride'] != H * W * Cout, len(levels) > 1), p['pixels']))
            if a['dbias'] is not None:
                c = _colsum_plan(B * H * W, Cout)
                out.append((('colsum', c['rows']), c['rpb']))
    return out


def _signature(kind, levels):
    """what a GPU case needs to repeat one recorded call: (kind, ksize, Cin, Cout, B, ((H, W) per level), prologue,
    epilogue, activation, x in a concatenated buffer, y (dy) in a concatenated buffer, dbias)"""
    a = levels[0]
    B, Cin, Cout, k = (a[f] for f in ('B', 'Cin', 'Cout', 'ksize'))
    hw = tuple((lv['H'], lv['W']) for lv in levels)
    pro = tuple(f for f in PROLOGUE if a[f] is not None)
    if kind != 'wgrad':
        epi = tuple(f for f in EPILOGUE if a[f] is not None)
        xs = any(lv['x_bstride'] != lv['H'] * lv['W'] * Cin for lv in levels)
        ys = any(lv['y_bstride'] != lv['H'] * lv['W'] * Cout for lv in levels)
        return (kind, k, Cin, Cout, B, hw, pro, epi, ACTS[a['act']], xs, ys, False)
    ys = any(lv['dy_bstride'] != lv['H'] * lv['W'] * Cout for lv in levels)
    return (kind, k, Cin, Cout, B, hw, pro, (), 'none', False, ys, a['dbias'] is not None)


def _sig_levels(sig):
    """level argument dicts of a signature, as _classes reads them (a concatenated buffer holds all levels)"""
    kind, k, Cin, Cout, B, hw, pro, epi, act, xs, ys, dbias = sig
    tot = sum(h * w for h, w in hw)
    out = []
    for h, w in hw:
        a = {f: (1 if f in pro or f in epi else None) for f in PROLOGUE + EPILOGUE}
        a.update(B=B, H=h, W=w, Cin=Cin, Cout=Cout, ksize=k, act={v: n for n, v in ACTS.items()}[act],
                 x_bstride=(tot if xs else h * w) * Cin, y_bstride=(tot if ys else h * w) * Cout,
                 dy_bstride=(tot if ys else h * w) * Cout, dbias=1 if dbias else None)
        out.append(a)
    return out


# ------------------------------------------------------------------------------------------------
# the recorded traces
# ------------------------------------------------------------------------------------------------

CONV_CALLS = {'effdet_conv2d': 'conv', 'effdet_conv2d_multi': 'conv', 'effdet_conv2d_wgrad': 'wgrad',
              'effdet_conv2d_wgrad_multi': 'wgrad'}


def _record_traces():
    """{config: [(fwd | dgrad | wgrad, [level argument dicts])]} of one fp32-mode step of bench.CONFIGS d0 and d4
    (the second, steady-state train step) and of the d7 forward (backbone + BiFPN + head; detection reads device values
    on the host and is left out).  Nothing is computed: the C ABI is replaced by the host-trace Recorder."""
    import __graft_entry__ as entry
    entry.build()
    from bench import CONFIGS
    from models import EfficientDet, _native as N, _ops
    rec = Recorder()
    traces = {}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(N, 'f32', rec.f32)
        mp.setattr(N, 'ptr', rec.ptr)
        mp.setattr(N, 'call', rec.call)
        mp.setattr(_ops, 'check_cuda_f32', lambda x, what: None)
        mp.setattr(_ops, '_cache', {})
        mp.setattr(_ops, 'PRECISION', 'fp32')
        for name in ('d0', 'd4', 'd7'):
            c = CONFIGS[name]
            cfg = O.make_config(c['net'], c['K'], c['W'], c['D'])
            m = EfficientDet(num_classes=c['K'], network=c['net'], D_bifpn=c['D'], W_bifpn=c['W'], is_training=True)
            m.load_state_dict(O.init_state_dict(cfg, seed=0))
            images, ann = O.synthetic_batch(c['bs'], size=c['size'], num_classes=c['K'], seed=3)
            if c['mode'] == 'train':
                m.train()
                m.is_training = True
                m.freeze_bn()
                for _ in range(2):
                    for p in m.parameters():
                        p.grad = None
                    start = len(rec.calls)
                    cl, rl = m([images, ann])
                    back = len(rec.calls)
                    (cl.mean() + rl.mean()).backward()
            else:
                m.eval()
                start = len(rec.calls)
                with torch.no_grad():
                    m.bbox_head.forward_concat_nhwc(m.extract_feat_nhwc(images))
                back = len(rec.calls)
            # a conv call of the backward pass is a data gradient (the rotated, transposed pack)
            traces[name] = [(CONV_CALLS[n] if CONV_CALLS[n] == 'wgrad' else 'fwd' if i < back else 'dgrad',
                             s[0] if isinstance(s[0], list) else [s[0]])
                            for i, (n, s) in enumerate(rec.calls) if i >= start and n in CONV_CALLS]
            del m, images, ann
    return traces


# ------------------------------------------------------------------------------------------------
# the cases: (config, signature), every one a call of its config's trace (test_cases_are_recorded_calls)
# ------------------------------------------------------------------------------------------------

CASES = [
    # d0 class conv, all levels, sigmoid into the concatenated buffer
    ('d0', ('fwd', 3, 256, 720, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), ('bias',), 'sigmoid', False,
            True, False)),
    # its data gradient 720 -> 256 at the buffer's batch stride, ReLU mask (405 K-steps)
    ('d0', ('dgrad', 3, 720, 256, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), ('mask_src',), 'none',
            True, False, False)),
    # its weight and bias gradients: 32 768 pixels per CTA
    ('d0', ('wgrad', 3, 256, 720, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), (), 'none', False, True,
            True)),
    # d0 box conv (36 outputs on the 64-column tile)
    ('d0', ('fwd', 3, 256, 36, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), ('bias',), 'none', False,
            True, False)),
    # d0 BiFPN node conv, W 64 (64-column tile)
    ('d0', ('fwd', 3, 64, 64, 32, ((64, 64),), (), ('bias',), 'none', False, False, False)),
    # d4 BiFPN node conv, W 224 (32-column tile)
    ('d4', ('fwd', 3, 224, 224, 4, ((128, 128),), (), ('bias',), 'none', False, False, False)),
    # d7 BiFPN node conv, W 384 (128-column tile)
    ('d7', ('fwd', 3, 384, 384, 1, ((192, 192),), (), ('bias',), 'none', False, False, False)),
    # d0 block-1 expand at 256^2: forward raw (the largest igemm grid)
    ('d0', ('fwd', 1, 16, 96, 32, ((256, 256),), (), (), 'none', False, False, False)),
    # its data gradient
    ('d0', ('dgrad', 1, 96, 16, 32, ((256, 256),), (), (), 'none', False, False, False)),
    # d0 block-2 expand data gradient with the residual
    ('d0', ('dgrad', 1, 144, 24, 32, ((128, 128),), (), ('residual',), 'none', False, False, False)),
    # d0 block-1 expand weight gradient <32,128,4,4>
    ('d0', ('wgrad', 1, 16, 96, 32, ((256, 256),), (), (), 'none', False, False, False)),
    # d0 block-2 project conv, full prologue and epilogue
    ('d0', ('fwd', 1, 144, 24, 32, ((128, 128),), ('in_scale', 'a_scale'), ('z', 'scale', 'row_scale', 'residual'),
            'none', False, False, False)),
    # its weight gradient <128,32,4,4> with the same prologue
    ('d0', ('wgrad', 1, 144, 24, 32, ((128, 128),), ('in_scale', 'a_scale'), (), 'none', False, False, False)),
    # d0 BiFPN lateral with bias
    ('d0', ('fwd', 1, 40, 64, 32, ((64, 64),), (), ('bias',), 'none', False, False, False)),
    # its weight and bias gradients
    ('d0', ('wgrad', 1, 40, 64, 32, ((64, 64),), (), (), 'none', False, False, True)),
    # d4 class conv weight gradient: 16 384 pixels per CTA
    ('d4', ('wgrad', 3, 256, 720, 4, ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8)), (), (), 'none', False, True,
            True)),
    # the cheapest recorded call of each plan class not reached above
    ('d4', ('wgrad', 1, 448, 224, 4, ((8, 8),), (), (), 'none', False, False, True)),
    ('d4', ('wgrad', 3, 256, 36, 4, ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8)), (), (), 'none', False, True,
            True)),
    ('d7', ('fwd', 3, 256, 256, 1, ((192, 192), (96, 96), (48, 48), (24, 24), (12, 12)), (), ('bias',), 'relu',
            False, False, False)),
    ('d0', ('dgrad', 1, 64, 320, 32, ((4, 4),), (), (), 'none', False, False, False)),
    ('d0', ('wgrad', 3, 64, 64, 32, ((4, 4),), (), (), 'none', False, False, True)),
    ('d0', ('dgrad', 3, 64, 64, 32, ((4, 4),), (), (), 'none', False, False, False)),
    ('d4', ('fwd', 1, 448, 224, 4, ((8, 8),), (), ('bias',), 'none', False, False, False)),
    ('d7', ('fwd', 1, 576, 384, 1, ((12, 12),), (), ('bias',), 'none', False, False, False)),
    ('d0', ('dgrad', 1, 64, 112, 32, ((16, 16),), (), (), 'none', False, False, False)),
    ('d4', ('wgrad', 3, 224, 224, 4, ((8, 8),), (), (), 'none', False, False, True)),
    ('d4', ('dgrad', 3, 224, 224, 4, ((8, 8),), (), (), 'none', False, False, False)),
    ('d7', ('fwd', 1, 2064, 576, 1, ((12, 12),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d7', ('fwd', 1, 200, 384, 1, ((48, 48),), (), ('bias',), 'none', False, False, False)),
    ('d4', ('fwd', 1, 1632, 448, 4, ((8, 8),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d4', ('wgrad', 1, 1632, 448, 4, ((8, 8),), ('in_scale', 'a_scale'), (), 'none', False, False, False)),
    ('d0', ('dgrad', 1, 320, 1152, 32, ((4, 4),), (), (), 'none', False, False, False)),
    ('d7', ('fwd', 3, 384, 384, 1, ((12, 12),), (), ('bias',), 'none', False, False, False)),
    ('d7', ('fwd', 1, 1200, 344, 1, ((24, 24),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d4', ('fwd', 1, 960, 272, 4, ((16, 16),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d7', ('fwd', 1, 576, 3456, 1, ((12, 12),), (), (), 'none', False, False, False)),
    ('d7', ('fwd', 1, 3456, 576, 1, ((12, 12),), ('in_scale', 'a_scale'), ('z', 'scale', 'residual'), 'none', False,
            False, False)),
    ('d4', ('fwd', 1, 2688, 448, 4, ((8, 8),), ('in_scale', 'a_scale'), ('z', 'scale', 'row_scale', 'residual'),
            'none', False, False, False)),
    ('d4', ('dgrad', 1, 2688, 448, 4, ((8, 8),), (), ('residual',), 'none', False, False, False)),
    ('d0', ('dgrad', 1, 64, 40, 32, ((64, 64),), (), (), 'none', False, False, False)),
    ('d7', ('fwd', 1, 344, 2064, 1, ((24, 24),), (), (), 'none', False, False, False)),
    ('d7', ('fwd', 1, 2064, 344, 1, ((24, 24),), ('in_scale', 'a_scale'), ('z', 'scale', 'residual'), 'none', False,
            False, False)),
    ('d0', ('fwd', 1, 480, 112, 32, ((16, 16),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d0', ('wgrad', 1, 480, 112, 32, ((16, 16),), ('in_scale', 'a_scale'), (), 'none', False, False, False)),
    ('d4', ('fwd', 1, 672, 160, 4, ((32, 32),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d7', ('fwd', 1, 1200, 200, 1, ((48, 48),), ('in_scale', 'a_scale'), ('z', 'scale', 'residual'), 'none', False,
            False, False)),
    ('d4', ('wgrad', 1, 24, 24, 4, ((512, 512),), ('in_scale', 'a_scale'), (), 'none', False, False, False)),
    ('d7', ('fwd', 1, 32, 32, 1, ((768, 768),), ('in_scale', 'a_scale'), ('z', 'scale', 'residual'), 'none', False,
            False, False)),
    ('d0', ('fwd', 1, 672, 112, 32, ((16, 16),), ('in_scale', 'a_scale'), ('z', 'scale', 'row_scale', 'residual'),
            'none', False, False, False)),
    ('d0', ('dgrad', 1, 672, 112, 32, ((16, 16),), (), ('residual',), 'none', False, False, False)),
    ('d4', ('fwd', 1, 960, 160, 4, ((32, 32),), ('in_scale', 'a_scale'), ('z', 'scale', 'row_scale', 'residual'),
            'none', False, False, False)),
    ('d4', ('dgrad', 1, 960, 160, 4, ((32, 32),), (), ('residual',), 'none', False, False, False)),
    ('d4', ('fwd', 1, 192, 56, 4, ((128, 128),), ('in_scale', 'a_scale'), ('z', 'scale'), 'none', False, False, False)),
    ('d4', ('fwd', 1, 336, 56, 4, ((128, 128),), ('in_scale', 'a_scale'), ('z', 'scale', 'row_scale', 'residual'),
            'none', False, False, False)),
    ('d4', ('dgrad', 1, 336, 56, 4, ((128, 128),), (), ('residual',), 'none', False, False, False)),
    ('d7', ('fwd', 1, 240, 40, 1, ((384, 384),), ('in_scale', 'a_scale'), ('z', 'scale', 'residual'), 'none', False,
            False, False)),
    ('d7', ('fwd', 3, 256, 36, 1, ((192, 192), (96, 96), (48, 48), (24, 24), (12, 12)), (), ('bias',), 'none', False,
            True, False)),
    ('d0', ('wgrad', 3, 64, 256, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), (), 'none', False, False,
            True)),
    ('d0', ('dgrad', 3, 256, 64, 32, ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4)), (), ('residual',), 'none',
            False, False, False)),
    ('d4', ('wgrad', 3, 224, 256, 4, ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8)), (), (), 'none', False,
            False, True)),
    ('d4', ('dgrad', 3, 256, 224, 4, ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8)), (), ('residual',), 'none',
            False, False, False)),
    ('d4', ('dgrad', 3, 256, 256, 4, ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8)), (), ('mask_src',), 'none',
            False, False, False)),
    ('d7', ('fwd', 3, 256, 720, 1, ((192, 192), (96, 96), (48, 48), (24, 24), (12, 12)), (), ('bias',), 'sigmoid',
            False, True, False)),
]


def _case_id(case):
    cfg, (kind, k, Cin, Cout, B, hw) = case[0], case[1][:6]
    return '%s-%s-k%d-%d-%d-B%d-%dx%d%s' % (cfg, kind, k, Cin, Cout, B, hw[0][0], hw[0][1],
                                           '-L%d' % len(hw) if len(hw) > 1 else '')


def _case_classes(case):
    return {c for c, _ in _classes(case[1][0], _sig_levels(case[1]))}


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def traces():
    return _record_traces()


def test_mirrors():
    """the launchers' arithmetic on the figures that motivated the cases (132 SMs).  The head's feature width is 256
    at every config, so the class conv is 256 -> 720 and its weight gradient takes <128,128,8,8>"""
    d0 = [(64, 64), (32, 32), (16, 16), (8, 8), (4, 4)]
    p = _wgrad_plan(32, 64, 64, 256, 720, 3)                 # d0 class conv, P3
    assert (p['inst'], p['ctiles'], p['ntiles'], p['nchunks'], p['splits'], p['pixels'], p['grid']) == \
        ((128, 128, 8, 8), 2, 6, 8192, 4, 32768, (12, 9, 4))
    p = _wgrad_plan(4, 128, 128, 256, 720, 3)                # d4 class conv, P3
    assert (p['inst'], p['splits'], p['pixels'], p['grid']) == ((128, 128, 8, 8), 4, 16384, (12, 9, 4))
    assert [_wgrad_plan(32, h, w, 256, 720, 3)['pixels'] for h, w in d0] == [32768, 8192, 2048, 512, 256]
    # the four instantiations
    assert _wgrad_plan(32, 256, 256, 16, 96, 1)['inst'] == (32, 128, 4, 4)
    assert _wgrad_plan(32, 128, 128, 144, 24, 1)['inst'] == (128, 32, 4, 4)
    assert _wgrad_plan(32, 64, 64, 40, 64, 1)['inst'] == (64, 64, 4, 4)
    # the class conv: 720 outputs on the 32-column tile, 23 n-tiles, the last one half full; its data gradient is the
    # longest reduction, 9 taps x 45 slices of 16 channels
    c = _igemm_plan(32, 64, 64, 256, 720, 3)
    assert (c['BN'], c['grid'], c['tail'], c['kernel']) == (32, (1024, 23, 1), 16, 'conv_igemm_kernel<32,4>(')
    assert _igemm_plan(32, 64, 64, 720, 256, 3)['ksteps'] == 405
    b = _igemm_plan(32, 64, 64, 256, 36, 3)                  # box conv: 64-column tile, 28 padded columns
    assert (b['BN'], b['grid'][1], b['tail']) == (64, 1, 36)
    assert [_igemm_plan(1, 8, 8, w, w, 3)['BN'] for w in (64, 224, 384)] == [64, 32, 128]
    assert _igemm_plan(1, 4, 4, 64, 128, 3)['BN'] == 128   # a tie goes to the wider tile
    # column sums: one row lane for 720 columns, 16 for 64; rows per block from four waves, at least 8 iterations
    assert _colsum_plan(32 * 4096, 720) == dict(rows=1, rpb=249, grid=(527, 1, 1))
    assert _colsum_plan(32 * 16, 64) == dict(rows=16, rpb=128, grid=(4, 1, 1))


def test_cases_are_recorded_calls(traces):
    """every case repeats a call of its config's trace, and the level dicts it is built from sort into the classes the
    recorded call does"""
    recorded = {cfg: {_signature(k, lv): lv for k, lv in calls} for cfg, calls in traces.items()}
    ids = [_case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids)
    for cfg, sig in CASES:
        assert sig in recorded[cfg], (cfg, sig)
        assert _case_classes((cfg, sig)) == {c for c, _ in _classes(sig[0], recorded[cfg][sig])}, (cfg, sig)


def test_traces_take_the_exact_fp32_route_and_cases_cover_them(traces):
    """every level of every recorded conv call takes the exact-fp32 route, and CASES reach every plan class of the
    three traces, their longest weight-gradient accumulation, their longest reduction and their largest igemm grid"""
    covered = set().union(*(_case_classes(c) for c in CASES))
    print()
    print('%-6s %5s  %-120s %s' % ('config', 'count', 'class', 'worst (grid CTAs | pixels per CTA | rows per block)'))
    worst_px, worst_ks, worst_grid = {}, 0, 0
    for cfg, calls in traces.items():
        assert calls, cfg
        count, worst = collections.Counter(), {}
        for kind, levels in calls:
            for a in levels:
                if kind == 'wgrad':
                    assert a['precision'] == 0 and a['dy_planes'] is None and a['x_planes'] is None, a
                else:
                    assert a['w_tc'] is None and a['tc_single'] == 0 and a['x_planes'] is None, a
                    p = _igemm_plan(a['B'], a['H'], a['W'], a['Cin'], a['Cout'], a['ksize'])
                    worst_ks = max(worst_ks, p['ksteps'])
            for cl, fig in _classes(kind, levels):
                count[cl] += 1
                worst[cl] = max(worst.get(cl, 0), fig)
                if cl[0] == 'wgrad':
                    worst_px[cfg] = max(worst_px.get(cfg, 0), fig)
                elif cl[0] == 'igemm':
                    worst_grid = max(worst_grid, fig)
        for cl in sorted(count, key=str):
            print('%-6s %5d  %-120s %d' % (cfg, count[cl], cl, worst[cl]))
        missing = set(count) - covered
        assert not missing, (cfg, missing)
    assert worst_px == {'d0': 32768, 'd4': 16384}, worst_px
    assert worst_ks == 405
    case_px = max(f for c in CASES for cl, f in _classes(c[1][0], _sig_levels(c[1])) if cl[0] == 'wgrad')
    case_ks = max(_igemm_plan(a['B'], a['H'], a['W'], a['Cin'], a['Cout'], a['ksize'])['ksteps']
                  for c in CASES if c[1][0] != 'wgrad' for a in _sig_levels(c[1]))
    case_grid = max(f for c in CASES for cl, f in _classes(c[1][0], _sig_levels(c[1])) if cl[0] == 'igemm')
    print('longest accumulation %d pixels per CTA, longest reduction %d K-steps, largest igemm grid %d CTAs'
          % (case_px, case_ks, case_grid))
    assert (case_px, case_ks, case_grid) == (32768, 405, worst_grid)


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _dev():
    return torch.device('cuda:0')


def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


def _buffer(hw, B, C, concat, fill=float('nan')):
    """one fp32 buffer holding every level, GUARD NaN elements after it: the concatenated [B, sum(HW) * C] layout of
    RetinaHeadFn (concat) or dense [B, H, W, C] maps one after the other -> (buffer, elements in use, per level
    (pointer, batch stride, [B, H, W, C] view))"""
    tot = sum(h * w for h, w in hw)
    n = B * tot * C
    buf = torch.full((n + GUARD,), fill, device=_dev())
    buf[n:] = float('nan')
    lv, off = [], 0
    for h, w in hw:
        if concat:
            v = buf[:n].view(B, tot * C)[:, off * C:(off + h * w) * C].view(B, h, w, C)
            lv.append((buf.data_ptr() + 4 * off * C, tot * C, v))
            off += h * w
        else:
            v = buf[off:off + B * h * w * C].view(B, h, w, C)
            lv.append((buf.data_ptr() + 4 * off, h * w * C, v))
            off += B * h * w * C
    return buf, n, lv


def _check_written(buf, n, what):
    assert not torch.isnan(buf[:n]).any(), ('%s: an output element was not written' % what)
    assert torch.isnan(buf[n:]).all(), ('%s: written past the end of the output' % what)


def _setup(case):
    """the operands of a case, and launch() which runs the call once (-> its outputs) as the product makes it"""
    from models import _native as N, _ops as ops
    cfg, sig = case
    kind, k, Cin, Cout, B, hw, pro, epi, act, xs, ys, dbias = sig
    g = torch.Generator(device=_dev()).manual_seed(sum(map(ord, _case_id(case))))

    def randn(*shape):
        return torch.randn(*shape, generator=g, device=_dev())
    s = dict(case=case, kind=kind, k=k, Cin=Cin, Cout=Cout, B=B, hw=hw, epi=epi, act=act, xs=xs, ys=ys)
    s['in_scale'] = 1 + 0.25 * randn(Cin) if 'in_scale' in pro else None
    s['in_shift'] = 0.25 * randn(Cin) if 'in_scale' in pro else None
    s['a_scale'] = torch.sigmoid(randn(B, Cin)) if 'a_scale' in pro else None
    if kind == 'wgrad':
        _, _, s['x'] = _buffer(hw, B, Cin, False, 0.0)
        _, _, s['dy'] = _buffer(hw, B, Cout, ys, 0.0)
        for (_, _, x), (_, _, d) in zip(s['x'], s['dy']):
            x.copy_(randn(*x.shape))
            d.copy_(randn(*d.shape) + 0.5)     # gradients with a mean, as the focal loss's class gradients have
        s['shape'] = (Cout, Cin, k, k)

        def launch(dw, db):
            arr = (N.WgradArgs * len(hw))()
            for i, ((h, w), (xp, xbs, _), (dp, dbs, _)) in enumerate(zip(hw, s['x'], s['dy'])):
                arr[i] = N.WgradArgs(x=xp, x_bstride=xbs, dy=dp, dy_bstride=dbs, dw=N.f32(dw), dbias=N.f32(db),
                                     a_scale=N.f32(s['a_scale']), B=B, H=h, W=w, Cin=Cin, Cout=Cout, ksize=k,
                                     precision=0, in_scale=N.f32(s['in_scale']), in_shift=N.f32(s['in_shift']))
            if len(hw) == 1:
                N.call('effdet_conv2d_wgrad', dw, arr[0])
            else:
                N.call('effdet_conv2d_wgrad_multi', dw, arr, len(hw))
        s['launch'] = launch
        s['dbias'] = dbias
        return s
    _, _, s['x'] = _buffer(hw, B, Cin, xs, 0.0)
    for _, _, x in s['x']:
        x.copy_(randn(*x.shape))
    # forward: OIHW [Cout, Cin]; data gradient: the forward layer's [Cin, Cout] weight on its rotated, transposed pack
    oi = (Cout, Cin) if kind == 'fwd' else (Cin, Cout)
    w = randn(*oi, k, k) / math.sqrt(k * k * oi[1])
    s['w'] = w
    packs = ops.pack_conv(w)
    wp = packs[0] if kind == 'fwd' else packs[1]
    s['bias'] = 0.1 * randn(Cout) if 'bias' in epi else None
    s['scale'] = 1 + 0.25 * randn(Cout) if 'scale' in epi else None
    s['shift'] = 0.25 * randn(Cout) if 'scale' in epi else None
    if 'row_scale' in epi:
        s['row_scale'] = torch.full((B,), 1.25, device=_dev())
        s['row_scale'][1 % B] = 0.0                          # one image dropped by drop-connect
    else:
        s['row_scale'] = None
    s['residual'] = _buffer(hw, B, Cout, False, 0.0)[2] if 'residual' in epi else None
    s['mask'] = _buffer(hw, B, Cout, False, 0.0)[2] if 'mask_src' in epi else None
    for t in (s['residual'] or []) + (s['mask'] or []):
        t[2].copy_(randn(*t[2].shape))
    actn = {n: v for v, n in ACTS.items()}[act]

    def launch():
        ybuf, yn, ylv = _buffer(hw, B, Cout, ys)
        zbuf, zn, zlv = _buffer(hw, B, Cout, False) if 'z' in epi else (None, 0, [(None, 0, None)] * len(hw))
        arr = (N.ConvArgs * len(hw))()
        for i, (h, w_) in enumerate(hw):
            r = s['residual'][i] if s['residual'] else (None, 0, None)
            m = s['mask'][i] if s['mask'] else (None, 0, None)
            arr[i] = N.ConvArgs(x=s['x'][i][0], x_bstride=s['x'][i][1], w=N.f32(wp), y=ylv[i][0], y_bstride=ylv[i][1],
                                z=zlv[i][0], bias=N.f32(s['bias']), scale=N.f32(s['scale']), shift=N.f32(s['shift']),
                                a_scale=N.f32(s['a_scale']), row_scale=N.f32(s['row_scale']), residual=r[0],
                                r_bstride=r[1], mask_src=m[0], m_bstride=m[1], B=B, H=h, W=w_, Cin=Cin, Cout=Cout,
                                ksize=k, act=actn, in_scale=N.f32(s['in_scale']), in_shift=N.f32(s['in_shift']))
        if len(hw) == 1:
            N.call('effdet_conv2d', ybuf, arr[0])
        else:
            N.call('effdet_conv2d_multi', ybuf, arr, len(hw))
        return dict(y=(ybuf, yn, [v for _, _, v in ylv]),
                    z=(zbuf, zn, [v for _, _, v in zlv]) if zbuf is not None else None)
    s['launch'] = launch
    return s


def _expected_launches(case, sms):
    """[(kernel name, grid)] of one call: an igemm launch per level; a weight-gradient launch per level, each followed
    by its column sum when the call has a dbias"""
    kind, k, Cin, Cout, B, hw = case[1][:6]
    out = []
    for h, w in hw:
        if kind == 'wgrad':
            p = _wgrad_plan(B, h, w, Cin, Cout, k, sms)
            out.append((p['kernel'], p['grid']))
            if case[1][-1]:
                out.append(('colsum_kernel(', _colsum_plan(B * h * w, Cout, sms)['grid']))
        else:
            p = _igemm_plan(B, h, w, Cin, Cout, k)
            out.append((p['kernel'], p['grid']))
    return out


KERNELS = ('conv_igemm_kernel', 'conv_wgrad_kernel', 'colsum_kernel')


def _record_launches(out_dir):
    """run every case once under torch.profiler; write {case id: [(kernel name, grid)]} to out_dir/launches.json"""
    from torch.profiler import ProfilerActivity, profile
    out_dir = pathlib.Path(out_dir)
    rec = {}
    # the first profiler session of a process has come back without any CUDA activity: open one on a throw-away launch
    with profile(activities=[ProfilerActivity.CUDA]):
        torch.ones(1024, device=_dev()).add_(1)
        torch.cuda.synchronize()
    for case in CASES:
        s = _setup(case)
        if s['kind'] == 'wgrad':
            dw = torch.zeros(s['shape'], device=_dev())
            db = torch.zeros(s['Cout'], device=_dev()) if s['dbias'] else None
            fn = lambda: s['launch'](dw, db)                      # noqa: E731
        else:
            fn = s['launch']
        rec[_case_id(case)] = [t for t in _launches(fn, out_dir, '_kernel') if any(k in t[0] for k in KERNELS)]
        del s
        torch.cuda.empty_cache()
    with open(out_dir / 'launches.json', 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def launches(tmp_path_factory):
    """the kernel names and grids of every case, recorded by _record_launches in a fresh interpreter: a CUDA activity
    trace in a long test process can miss this library's kernels after some of the other tests have run"""
    out = tmp_path_factory.mktemp('exact_fp32_launches')
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    path = [here, os.path.join(repo, 'oracle'), os.path.join(repo, 'efficientdet.pytorch_b200'), repo]
    code = ('import sys; sys.path[:0] = %r; import test_exact_fp32_parity as T; T._record_launches(%r)'
            % (path, str(out)))
    subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], check=True, cwd=repo,
                   timeout=1800)
    with open(out / 'launches.json') as f:
        return {k: [(name, tuple(grid)) for name, grid in v] for k, v in json.load(f).items()}


# ------------------------------------------------------------------------------------------------
# float64 references and bounds
# ------------------------------------------------------------------------------------------------

def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _operand(s, x, b0):
    """the prologue operand swish(x * in_scale + in_shift) * a_scale in float64 from the fp32 x of images b0.. (NHWC),
    and the bound E_A of the kernel's own fp32 evaluation of it (None without a prologue)"""
    a, e = x.double(), None
    if s['in_scale'] is not None:
        v = a * s['in_scale'].double() + s['in_shift'].double()
        sg = torch.sigmoid(v)
        a = v * sg
        e = (a * (1 + v * (1 - sg))).abs() + 7 * a.abs()           # |v swish'(v)| + 7 |swish(v)|
    if s['a_scale'] is not None:
        gt = s['a_scale'][b0:b0 + x.shape[0]].double()[:, None, None, :]
        a = a * gt
        e = (0 if e is None else e * gt.abs()) + a.abs()
    return a, (None if e is None else e * (U * (1 + 1e-3)))


def _epilogue(s, lv, b0, acc, E):
    """the kernel's epilogue in its order on the fp64 accumulator and its bound (NHWC) -> {'y': (value, bound),
    'z': (value, bound) when the call stores z}"""
    v = acc
    if s.get('bias') is not None:
        v = v + s['bias'].double()
        E = E + U * v.abs()
    out = {'z': (v, E)} if 'z' in s['epi'] else {}
    if s.get('scale') is not None:
        sc = s['scale'].double()
        v = v * sc + s['shift'].double()
        E = sc.abs() * E + U * v.abs()
    if s['act'] == 'relu':
        v = torch.relu(v)
    elif s['act'] == 'sigmoid':
        v = torch.sigmoid(v)
        E = E / 4 + 6 * U * v
    elif s['act'] == 'swish':
        v = v * torch.sigmoid(v)
        E = 1.1 * E + 7 * U * v.abs()
    nb = acc.shape[0]
    if s.get('row_scale') is not None:
        r = s['row_scale'][b0:b0 + nb].double()[:, None, None, None]
        v = v * r
        E = r.abs() * E + U * v.abs()
    if s.get('residual') is not None:
        v = v + s['residual'][lv][2][b0:b0 + nb].double()
        E = E + U * v.abs()
    if s.get('mask') is not None:
        keep = s['mask'][lv][2][b0:b0 + nb] > 0
        v, E = v * keep, E * keep
    out['y'] = (v, E)
    return out


class _Stats:
    """per-element ratio |got - ref| / bound and norm-relative errors of one output: whole tensor, per image (dim 0)
    and per block of 64 channels (last dim)"""

    def __init__(self, name, C):
        self.name, self.worst, self.bad, self.where = name, 0.0, 0, None
        self.d2 = self.r2 = 0.0
        self.img = collections.defaultdict(lambda: [0.0, 0.0])
        self.blk = torch.zeros(2, _cdiv(C, 64), dtype=torch.float64)

    def add(self, got, ref, bound, b0=0, lv=0, images=True):
        diff = got.double() - ref
        over = diff.abs() > bound
        ratio = torch.where(bound > 0, diff.abs() / bound.clamp_min(1e-300), over.double())
        r = float(ratio.max())
        if r > self.worst:
            idx = [int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape)]
            self.where = (lv, b0 + idx[0], idx[1:], float(got[tuple(idx)]), float(ref[tuple(idx)]),
                          float(bound[tuple(idx)]))
            self.worst = r
        n = int(over.sum())
        if n and self.bad < 8:
            for idx in over.nonzero()[:8 - self.bad].tolist():
                print('    %s: over its bound at level %d, index %s: got %.9g, ref %.9g, bound %.3g'
                      % (self.name, lv, [b0 + idx[0]] + idx[1:], float(got[tuple(idx)]), float(ref[tuple(idx)]),
                         float(bound[tuple(idx)])))
        self.bad += n
        d2, r2 = diff.pow(2), ref.pow(2)
        self.d2 += float(d2.sum())
        self.r2 += float(r2.sum())
        if images:
            for i in range(got.shape[0]):
                self.img[b0 + i][0] += float(d2[i].sum())
                self.img[b0 + i][1] += float(r2[i].sum())
        C = got.shape[-1]
        pad = self.blk.shape[1] * 64 - C
        self.blk[0] += F.pad(d2.reshape(-1, C).sum(0), (0, pad)).view(-1, 64).sum(1).cpu()
        self.blk[1] += F.pad(r2.reshape(-1, C).sum(0), (0, pad)).view(-1, 64).sum(1).cpu()

    def norms(self):
        rel = lambda d, r: math.sqrt(d / r) if r > 0 else float(d > 0)       # noqa: E731
        tensor = rel(self.d2, self.r2)
        image = max([rel(d, r) for d, r in self.img.values() if r > 0] or [0.0])
        block = max(rel(float(d), float(r)) for d, r in self.blk.t())
        return tensor, image, block

    def check(self, tol=TOL_EXACT):
        tensor, image, block = self.norms()
        print('  %s: worst |got - ref| / bound %.3f at %s, %d over; rel err %.2e (bound %.0e), worst image %.2e, worst '
              '64-channel block %.2e (bound %.0e)' % (self.name, self.worst, self.where, self.bad, tensor, tol, image,
                                                       block, TOL_LOCAL))
        assert self.bad == 0 and self.worst < 1, (self.name, self.worst, self.where)
        assert tensor < tol and image < TOL_LOCAL and block < TOL_LOCAL, (self.name, tensor, image, block)


def _chunk(s, C):
    """images per reference chunk: about 2^26 elements of each fp64 temporary"""
    return max(1, 2 ** 26 // (sum(h * w for h, w in s['hw']) * C))


def _conv_ref(s, lv, b0, b1, w=None):
    """fp64 accumulator and its bound gamma_n (|A| (*) |W|) + E_A (*) |W| of level lv, images b0..b1 (NHWC)"""
    w = s['w'].double() if w is None else w
    x = s['x'][lv][2][b0:b1]
    a, ea = _operand(s, x, b0)
    conv = F.conv2d if s['kind'] == 'fwd' else F.conv_transpose2d
    pad = s['k'] // 2
    acc = conv(_nchw(a), w, padding=pad).permute(0, 2, 3, 1)
    bound = _gamma(s['k'] ** 2 * s['Cin']) * conv(_nchw(a.abs()), w.abs(), padding=pad).permute(0, 2, 3, 1)
    if ea is not None:
        bound = bound + conv(_nchw(ea), w.abs(), padding=pad).permute(0, 2, 3, 1)
    return acc, bound * (1 + 1e-3)


# ------------------------------------------------------------------------------------------------
# the GPU tests
# ------------------------------------------------------------------------------------------------

@pytest.fixture()
def ops():
    from models import _ops
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(_ops, 'PRECISION', 'fp32')
        yield _ops


def _check_launch(case, launches, sms):
    got, want = launches[_case_id(case)], _expected_launches(case, sms)
    for name, grid in got:
        print('  %s grid %s' % (name, grid))
    assert len(got) == len(want) and all(n in g[0] and grid == g[1] for (n, grid), g in zip(want, got)), (got, want)


def _conv_case(s):
    """the call once (and again: no atomics, the two must be bit-identical), checked element-wise and in norm against
    the fp64 reference image-chunk by image-chunk; control: the reference without the first 16 channels of the centre
    tap on the first chunk of the first level"""
    out = s['launch']()
    again = s['launch']()
    what = '%s %s k%d %d->%d B=%d %s' % (s['case'][0], s['kind'], s['k'], s['Cin'], s['Cout'], s['B'], s['hw'])
    for key in ('y', 'z'):
        if out[key] is not None:
            _check_written(out[key][0], out[key][1], what + ' ' + key)
            assert torch.equal(out[key][0][:out[key][1]], again[key][0][:again[key][1]]), (what, key, 'not repeatable')
    del again
    stats = {key: _Stats(key, s['Cout']) for key in ('y', 'z') if out[key] is not None}
    step = _chunk(s, max(s['Cin'], s['Cout']))
    ctrl = None
    for lv in range(len(s['hw'])):
        for b0 in range(0, s['B'], step):
            b1 = min(s['B'], b0 + step)
            acc, bound = _conv_ref(s, lv, b0, b1)
            ref = _epilogue(s, lv, b0, acc, bound)
            for key, st in stats.items():
                st.add(out[key][2][lv][b0:b1], ref[key][0], ref[key][1], b0, lv)
            if ctrl is None:
                k, t = s['k'], s['k'] ** 2 // 2
                w16 = torch.zeros_like(s['w'], dtype=torch.float64)
                sl = (slice(None), slice(0, 16)) if s['kind'] == 'fwd' else (slice(0, 16), slice(None))
                w16[sl + (t // k, t % k)] = s['w'][sl + (t // k, t % k)].double()
                part, _ = _conv_ref(s, lv, b0, b1, w16)
                miss = _epilogue(s, lv, b0, acc - part, bound)['y'][0]
                reached = miss != ref['y'][0]
                over = ((out['y'][2][lv][b0:b1].double() - miss).abs() > ref['y'][1]) & reached
                ctrl = (float(over.sum()) / max(1, int(reached.sum())), int(reached.sum()))
            del acc, bound, ref
    for st in stats.values():
        st.check()
    print('  control: without 16 channels of the centre tap, %.1f %% of the %d outputs it reaches are over their bound'
          % (100 * ctrl[0], ctrl[1]))
    assert ctrl[1] > 0 and ctrl[0] > 0.5, ctrl


def _wgrad_case(s, sms):
    """the call once into a non-zero dw (and dbias), checked element-wise, in norm and per tap against the fp64
    reference summed over image chunks; controls: the reference without the last 16-pixel chunk of each split of the
    first level, the bias reference without the first row block of colsum_kernel on that level"""
    k, Cin, Cout, B, hw = (s[f] for f in ('k', 'Cin', 'Cout', 'B', 'hw'))
    shape, pad = s['shape'], k // 2
    ref = torch.zeros(shape, dtype=torch.float64, device=_dev())
    absr, eab = torch.zeros_like(ref), torch.zeros_like(ref)
    dref = torch.zeros(Cout, dtype=torch.float64, device=_dev())
    dabs = torch.zeros_like(dref)
    step = _chunk(s, max(Cin, Cout))
    for lv in range(len(hw)):
        for b0 in range(0, B, step):
            x, d = s['x'][lv][2][b0:b0 + step], s['dy'][lv][2][b0:b0 + step].double()
            a, ea = _operand(s, x, b0)
            ref += torch.nn.grad.conv2d_weight(_nchw(a), shape, _nchw(d), padding=pad)
            absr += torch.nn.grad.conv2d_weight(_nchw(a.abs()), shape, _nchw(d.abs()), padding=pad)
            if ea is not None:
                eab += torch.nn.grad.conv2d_weight(_nchw(ea), shape, _nchw(d.abs()), padding=pad)
            dref += d.sum((0, 1, 2))
            dabs += d.abs().sum((0, 1, 2))
    g = torch.Generator(device=_dev()).manual_seed(7)
    dw0 = torch.randn(shape, generator=g, device=_dev()) * float(ref.std())
    db0 = torch.randn(Cout, generator=g, device=_dev()) * float(dref.pow(2).mean().sqrt())
    dw, db = dw0.clone(), db0.clone() if s['dbias'] else None
    s['launch'](dw, db)
    plans = [_wgrad_plan(B, h, w, Cin, Cout, k, sms) for h, w in hw]
    n = max(p['pixels'] for p in plans) + sum(p['splits'] for p in plans) + 1
    bound = (_gamma(n) * (absr + dw0.double().abs()) + eab) * (1 + 1e-3)
    what = '%s wgrad k%d %d->%d B=%d %s' % (s['case'][0], k, Cin, Cout, B, hw)
    print('  %s: pixels per CTA %s, splits %s, n = %d'
          % (what, [p['pixels'] for p in plans], [p['splits'] for p in plans], n))
    # element-wise on the whole dw, norms on dw - dw0 against the reference, per 64-output-channel block and per tap
    st = _Stats('dw', Cin)
    st.add(dw, dw0.double() + ref, bound, images=False)
    inc = dw.double() - dw0.double()
    rel = lambda a_, b_: float((a_ - b_).norm() / b_.norm())                 # noqa: E731
    st.d2, st.r2 = float((inc - ref).pow(2).sum()), float(ref.pow(2).sum())
    blocks = [rel(inc[n0:n0 + 64], ref[n0:n0 + 64]) for n0 in range(0, Cout, 64)]
    taps = [rel(inc[:, :, t // k, t % k], ref[:, :, t // k, t % k]) for t in range(k * k)]
    print('  dw: worst |got - ref| / bound %.3f at %s; rel err %.2e (bound %.0e), worst 64-output-channel block %.2e, '
          'worst tap %.2e (bound %.0e)' % (st.worst, st.where, math.sqrt(st.d2 / st.r2), TOL_EXACT, max(blocks),
                                            max(taps), TOL_LOCAL))
    assert st.bad == 0 and st.worst < 1, (st.worst, st.where)
    assert math.sqrt(st.d2 / st.r2) < TOL_EXACT and max(blocks) < TOL_LOCAL and max(taps) < TOL_LOCAL, (blocks, taps)
    # control: the last 16-pixel chunk of every split of the first level (one chunk alone is 3e-5 of a 2^19-pixel sum
    # with a mean, below what a norm bound of 1e-4 can see)
    h, w = hw[0]
    cps, nch = plans[0]['cps'], plans[0]['nchunks']
    last = torch.tensor([min((i + 1) * cps, nch) - 1 for i in range(plans[0]['splits'])], device=_dev())
    rows = (last[:, None] * KBK + torch.arange(KBK, device=_dev())).flatten()
    keep = torch.zeros(B * h * w, dtype=torch.bool, device=_dev())
    keep[rows[rows < B * h * w]] = True
    keep = keep.view(B, h, w, 1)
    part = torch.zeros_like(ref)
    for b0 in range(0, B, step):
        a, _ = _operand(s, s['x'][0][2][b0:b0 + step], b0)
        dm = s['dy'][0][2][b0:b0 + step].double() * keep[b0:b0 + step]
        part += torch.nn.grad.conv2d_weight(_nchw(a), shape, _nchw(dm), padding=pad)
    miss = max(rel(inc[:, :, t // k, t % k], (ref - part)[:, :, t // k, t % k]) for t in range(k * k))
    print('  control: dw without the last 16-pixel chunk of each split, worst tap %.2e' % miss)
    assert miss > TOL_LOCAL, miss
    if not s['dbias']:
        return
    cps = [_colsum_plan(B * h * w, Cout, sms) for h, w in hw]
    n = max(c['rpb'] for c in cps) + max(c['rows'] for c in cps) + sum(c['grid'][0] for c in cps) + 1
    bound = _gamma(n) * (dabs + db0.double().abs()) * (1 + 1e-3)
    sb = _Stats('dbias', Cout)
    sb.add(db[None], (db0.double() + dref)[None], bound[None], images=False)
    sb.d2, sb.r2 = float((db.double() - db0.double() - dref).pow(2).sum()), float(dref.pow(2).sum())
    print('  dbias: rows per block %s, n = %d; worst |got - ref| / bound %.3f, rel err %.2e (bound %.0e)'
          % ([c['rpb'] for c in cps], n, sb.worst, math.sqrt(sb.d2 / sb.r2), TOL_EXACT))
    assert sb.bad == 0 and sb.worst < 1 and math.sqrt(sb.d2 / sb.r2) < TOL_EXACT, (sb.worst, sb.where)
    first = s['dy'][0][2].reshape(B * h * w, Cout)[:cps[0]['rpb']].double().sum(0)
    over = float(((db.double() - (db0.double() + dref - first)).abs() > bound).double().mean())
    print('  control: dbias without the first row block, %.1f %% of the columns over their bound' % (100 * over))
    assert over > 0.5, over


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_exact_fp32_call(ops, case, launches):
    """one recorded fp32-mode call at its real shape: kernel names and grids as the mirrors have them, every output
    element within its derived bound of the fp64 reference, the norms within TOL_EXACT / TOL_LOCAL, and the
    kernel's negative control over its bound"""
    sms = _sms()
    _check_launch(case, launches, sms)
    s = _setup(case)
    if s['kind'] == 'wgrad':
        _wgrad_case(s, sms)
    else:
        _conv_case(s)
