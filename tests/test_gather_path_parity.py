"""Kernel-level fp64 parity of the gathering tensor-core path: the RetinaHead and BiFPN 3x3 layers at the D1-D3 and D5-D7
pyramids.

  conv_tc_kernel   forward and data gradient, fp32 activations gathered and split in the kernel, all levels in one launch
  wgrad_tc_kernel  weight gradient of each level without a TMA pixel box, one launch per level
  colsum_kernel    the bias gradient of those levels (conv_simt.cu)

The TMA-fed planes path needs a pixel box on every level (wg_geometry, conv_tc.cu: W <= 64 or W % 64 == 0, and a box of
a multiple of 16 pixels).  At the reference's input sizes only D0 and D4 have one everywhere:

  model  input  W_bifpn  P3..P7                 levels without a pixel box
  D1      640     88     80, 40, 20, 10, 5      all
  D2      768    112     96, 48, 24, 12, 6      96, 6
  D3      896    160     112, 56, 28, 14, 7     all
  D5     1280    288     160, 80, 40, 20, 10    all
  D6     1408    384     176, 88, 44, 22, 11    all
  D7     1536    384     192, 96, 48, 24, 12    96

so those heads and necks run conv_tc_kernel for every forward and data gradient, and in a weight gradient of D2 or D7 the
boxed levels go one at a time to wgrad_tc2_multi_kernel (bias gradient from to_planes_kernel) while the others go to
wgrad_tc_kernel + colsum_kernel, all adding into the same dw and dbias.  This file

  * mirrors conv_tc_launch and wgrad_tc_launch in Python (_conv_plan, _wgrad_plan) and checks, without a GPU, the table
    above against the library and that the GPU cases reach every plan class the native pyramids reach at B = 1..8
    (test_cases_reach_native_plan_classes);
  * runs every GPU call once under torch.profiler, in an interpreter of its own (the launches fixture), and compares
    kernel names and grids with the mirrors;
  * holds each call to a float64 reference of the same fp32 operands (F.conv2d, F.conv_transpose2d,
    torch.nn.grad.conv2d_weight, computed on the device), with negative controls that must fail their bounds.

Bounds (norm-relative error, as tests/test_planes_path_parity.py):
  TOL_TC    = 3e-5  each whole call
  TOL_LOCAL = 1e-4  each pyramid level of a forward or data-gradient output, each 64-output-channel x tap block of dw
  TOL_SUM   = 2e-5  dbias
Controls: the smallest level missing from the reference fails the per-level bound; one bf16 product per multiply-add
gives more than 3e-4; the dw reference without the first 64 chunks (4 096 pixels) of P3 fails the block bound; the
dbias reference without the last level fails TOL_SUM.

wgrad_tc_kernel takes BC = 256 input channels per CTA whenever Cin > 64, so at Cin 88-160 most of its wgmma work is on
zero-padded channels (one channel tile of 256 for 88, 112 or 160 channels).  That is a performance matter, not a
correctness one, and is left as it is.

Measured on an H100 80GB HBM3 at 700 W, the worst case of each test (whole call / worst level or block):
  forward, W -> W at 384 channels                       1.24e-5 / 1.24e-5
  data gradient, class conv 720 -> W                    2.26e-5 / 2.26e-5
  weight gradient, each level alone                     1.46e-5 / 1.48e-5
    of which P3 of d5 and d6, 58 and 61 chunks per CTA  1.38e-5 / 1.40e-5
  weight gradient, all levels in one call               1.36e-5 / 1.39e-5
  dbias                                                 2.05e-6
The forward and data-gradient error grows linearly with the reduction length 9 * Cin, by about 3.2e-9 per term over a
floor of about 3.5e-6, and is the same at every pyramid: 4.6e-6 at Cin 36, 5.2e-6 at 88, 9.7e-6 at 288, 1.25e-5 at 384,
2.26e-5 at 720.  The class conv's data gradient with 80 classes is therefore the case closest to TOL_TC (75 % of it);
this is the fp32 tensor-core accumulation, not a property of one pyramid or level.  The weakest controls: the
smallest level missing 1.0, one product per multiply-add 2.33e-3, dw without the first 64 chunks of P3 3.05e-1 (worst
block), dbias without the last level 4.63e-2."""
import json
import os
import pathlib
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from test_benchmark_plans import _launches
from test_planes_path_parity import (LEVEL_SETS, SINGLE_PASS_MIN, TOL_LOCAL, TOL_SUM, TOL_TC, WG_MAX_CHUNKS_PER_SPLIT,
                                     _block_errs, _box, _check, _check_dw, _single_pass, _split_plan)
from test_planes_path_parity import ops  # noqa: F401  (the bf16x3 fixture)

A = 9                           # anchors per pixel
K_CLS = 80                      # the class conv of 80 classes has 720 outputs
SMS = 132                       # H100 SXM: the SM count the native plans are walked at
GUARD = 4096                    # NaN elements after every output buffer
# (input size, W_bifpn) of the detectors whose head and neck run the gathering kernels (the reference's
# utils/config_eff.py); every size is a multiple of 128, so P3..P7 are size / 8 .. size / 128
PYRAMIDS = {'d1_640': (640, 88), 'd2_768': (768, 112), 'd3_896': (896, 160), 'd5_1280': (1280, 288),
            'd6_1408': (1408, 384), 'd7_1536': (1536, 384)}
NO_BOX = {'d1_640': 'all', 'd2_768': [(96, 96), (6, 6)], 'd3_896': 'all', 'd5_1280': 'all', 'd6_1408': 'all',
          'd7_1536': [(96, 96)]}
FWD_PYRAMIDS = ['d1_640', 'd3_896', 'd5_1280', 'd6_1408', 'd7_1536']


def _cdiv(a, b):
    return -(-a // b)


def _dev():
    return torch.device('cuda:0')


def _levels(geo):
    size = PYRAMIDS[geo][0]
    return [(size >> k, size >> k) for k in range(3, 8)]


def _channels(geo, layer):
    """(Cin, Cout) of the forward layer: head tower / BiFPN node W -> W, class conv W -> 720, box conv W -> 36"""
    w = PYRAMIDS[geo][1]
    return {'tower': (w, w), 'node': (w, w), 'first': (w, w), 'class': (w, A * K_CLS), 'box': (w, A * 4)}[layer]


# ------------------------------------------------------------------------------------------------
# mirrors of conv_tc_launch and wgrad_tc_launch (conv_tc.cu)
# ------------------------------------------------------------------------------------------------

def _conv_plan(levels, B, Cin, Cout):
    """one conv_tc_kernel launch over all levels: N tile, stages, K blocks per tap, first tile of each level, grid"""
    BN = 64 if Cout <= 64 else 128
    begins, tiles = [], 0
    for h, w in levels:
        begins.append(tiles)
        tiles += _cdiv(B * h * w, 128)
    return dict(BN=BN, stages=4 if BN == 64 else 3, kblocks=_cdiv(Cin, 64), tile_begin=begins, ntiles=_cdiv(Cout, BN),
                small=any(B * h * w < 128 for h, w in levels), grid=(tiles, _cdiv(Cout, BN), 1))


def _wgrad_plan(B, H, W, Cin, Cout, sms):
    """one wgrad_tc_kernel launch: channel tile BC, tiles, chunks of 64 pixels, chunks per split, splits, grid, and which
    rule set the split count ('cap': kWgMaxChunksPerSplit, 'min8': at least 8 chunks per split, 'one split', 'free':
    about two waves of CTAs)"""
    BC = 256 if Cin > 64 else 64
    ctiles, ntiles = _cdiv(Cin, BC), _cdiv(Cout, 128)
    nchunks = _cdiv(B * H * W, 64)
    waves = max(1, _cdiv(sms * 2, ctiles * ntiles * 9))
    splits = min(waves, _cdiv(nchunks, 8))
    capped = max(splits, _cdiv(nchunks, WG_MAX_CHUNKS_PER_SPLIT))
    cps = _cdiv(nchunks, capped)
    n = _cdiv(nchunks, cps)
    rule = 'one split' if n == 1 else 'cap' if capped > splits else 'min8' if splits < waves else 'free'
    return dict(BC=BC, stages=2 if BC == 256 else 4, ctiles=ctiles, ntiles=ntiles, nchunks=nchunks, cps=cps, splits=n,
                rule=rule, grid=(ctiles * ntiles, 9, n))


def _wgrad_launches(B, levels, Cin, Cout, sms):
    """[(kernel name, grid or None)] of one conv_wgrad_multi call on a pyramid with a level without a pixel box: one
    route per level"""
    out = []
    for h, w in levels:
        if _box(B, h, w) is None:
            p = _wgrad_plan(B, h, w, Cin, Cout, sms)
            out += [('wgrad_tc_kernel<%d,%d,3>(' % (p['BC'], p['stages']), p['grid']), ('colsum_kernel', None)]
        else:
            splits = _split_plan(B, [(h, w)], Cin, Cout, sms)[3]
            BC = 256 if Cin > 64 else 64
            out.append(('wgrad_tc2_multi_kernel<%d,%d,3>(' % (BC, 2 if BC == 256 else 4),
                        (_cdiv(Cin, BC) * _cdiv(Cout, 128), 9, splits)))
    return out


# ------------------------------------------------------------------------------------------------
# the GPU cases
# ------------------------------------------------------------------------------------------------

# forward: every FWD_PYRAMIDS pyramid x layer; B = 2 for the layers that write the concatenated [B, sum(HWA), width] outputs
# (the batch stride is not H*W*C there), B = 1 for the others
FWD_LAYERS = {'tower': 'relu', 'node': 'none', 'class': 'sigmoid', 'box': 'none'}
# data gradient: class 720 -> W and box 36 -> W read the concatenated gradient; tower W -> W with the ReLU mask; the first
# tower layer W -> W with the residual (the box tower adds the class tower's feature gradient)
DGRAD_LAYERS = ['class', 'box', 'tower', 'first']
# weight gradient: (pyramid, layer, B).  B = 1 reaches every plan class of its pyramid and layer (P3 binds the cap at
# d5, d6 and d7, the 8-chunk minimum at d1); B = 2 where the case stands for the batch stride of the concatenated dy,
# which the weight-gradient and column-sum kernels step by
WGRAD_CASES = [('d1_640', 'tower', 1), ('d1_640', 'class', 2), ('d1_640', 'box', 2),
               ('d2_768', 'tower', 1), ('d2_768', 'class', 1), ('d2_768', 'box', 2),
               ('d3_896', 'tower', 1), ('d3_896', 'class', 1), ('d3_896', 'box', 1),
               ('d5_1280', 'tower', 1), ('d5_1280', 'class', 1), ('d5_1280', 'box', 1),
               ('d6_1408', 'tower', 1), ('d6_1408', 'class', 1), ('d6_1408', 'box', 1),
               ('d7_1536', 'tower', 1), ('d7_1536', 'class', 1), ('d7_1536', 'box', 1)]


def _head(layer):
    return layer in ('class', 'box')


def _fwd_batch(layer):
    return 2 if _head(layer) else 1


def _dgrad_batch(layer):
    return 2 if _head(layer) else 1


def _conv_features(plan):
    f = {('tile', plan['BN'], plan['ntiles']), ('kblocks', plan['kblocks'])}
    if plan['small']:
        f.add('level with M < 128')
    return f


def _wgrad_features(p):
    return {p['rule'], ('ctiles', p['ctiles']), ('ntiles', p['ntiles'])}


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_routing_table():
    """the table of the docstring: which levels have a TMA pixel box, from the library's effdet_wgrad_tc_geometry_ok and
    from the Python mirror _box, at B = 1..8; D0 and D4 have one on every level; the D7 pyramid is bench.py's d7"""
    import __graft_entry__ as entry
    entry.build()
    from models import _native as N
    from bench import CONFIGS
    lib = N.load()
    for geo in PYRAMIDS:
        levels = _levels(geo)
        want = set(levels) if NO_BOX[geo] == 'all' else set(NO_BOX[geo])
        for B in range(1, 9):
            for h, w in levels:
                assert bool(lib.effdet_wgrad_tc_geometry_ok(B, h, w)) == (_box(B, h, w) is not None), (geo, B, h, w)
            assert {lv for lv in levels if _box(B, *lv) is None} == want, (geo, B)
    for geo in ('d0_512', 'd4_1024'):
        for B in range(1, 9):
            assert all(lib.effdet_wgrad_tc_geometry_ok(B, h, w) for h, w in LEVEL_SETS[geo]), (geo, B)
    d7 = CONFIGS['d7']
    assert (d7['size'], d7['W']) == PYRAMIDS['d7_1536'] and _levels('d7_1536')[-1] == (12, 12)
    assert [lv for lv, _ in _levels('d1_640')] == [80, 40, 20, 10, 5]


def test_mirrors():
    """the launchers' arithmetic on the figures that motivated the cases (132 SMs)"""
    # tower P3 at B = 1: the cap of 64 chunks per CTA binds at d5 and d6 (d7's P3 has a pixel box: the TMA-fed kernel,
    # whose launcher caps the chunks per CTA the same way, takes it; its 96x96 level gets about two waves)
    p5, p6 = (_wgrad_plan(1, PYRAMIDS[g][0] >> 3, PYRAMIDS[g][0] >> 3, PYRAMIDS[g][1], PYRAMIDS[g][1], SMS)
              for g in ('d5_1280', 'd6_1408'))
    assert (p5['rule'], p5['nchunks'], p5['cps'], p5['splits'], p5['grid']) == ('cap', 400, 58, 7, (6, 9, 7))
    assert (p6['rule'], p6['nchunks'], p6['cps'], p6['splits']) == ('cap', 484, 61, 8)
    p7 = _wgrad_plan(1, 96, 96, 384, 384, SMS)
    assert (p7['rule'], p7['nchunks'], p7['cps'], p7['splits']) == ('free', 144, 29, 5)
    assert _split_plan(1, [(192, 192)], 384, 384, SMS)[1:] == (576, 64, 9)
    # ... the 8-chunk minimum at d1, and P7 takes one split
    p1 = _wgrad_plan(1, 80, 80, 88, 88, SMS)
    assert (p1['rule'], p1['nchunks'], p1['cps'], p1['splits'], p1['grid']) == ('min8', 100, 8, 13, (1, 9, 13))
    assert _wgrad_plan(1, 5, 5, 88, 88, SMS)['rule'] == 'one split'
    # the class conv of d1 at B = 2: about two waves of CTAs
    pc = _wgrad_plan(2, 80, 80, 88, 720, SMS)
    assert (pc['rule'], pc['cps'], pc['splits'], pc['grid']) == ('free', 40, 5, (6, 9, 5))
    # the class conv's forward at d7, B = 2: 720 outputs in six tiles of 128 (the last 80 wide), 6 K blocks
    c = _conv_plan(_levels('d7_1536'), 2, 384, 720)
    assert (c['BN'], c['stages'], c['kblocks'], c['ntiles'], c['grid']) == (128, 3, 6, 6, (768, 6, 1))
    assert c['tile_begin'] == [0, 576, 720, 756, 765]
    # its data gradient: 720 -> 384, 12 K blocks, the last one 16 channels of data; the box conv's: one K block
    assert _conv_plan(_levels('d7_1536'), 2, 720, 384)['kblocks'] == 12
    b = _conv_plan(_levels('d1_640'), 1, 36, 88)
    assert (b['kblocks'], b['BN'], b['small']) == (1, 128, True)
    assert _conv_plan(_levels('d1_640'), 2, 88, 36)['BN'] == 64
    # a D2 weight gradient mixes routes
    names = [n for n, _ in _wgrad_launches(1, _levels('d2_768'), 112, 112, SMS)]
    assert names == ['wgrad_tc_kernel<256,2,3>(', 'colsum_kernel'] + ['wgrad_tc2_multi_kernel<256,2,3>('] * 3 + \
        ['wgrad_tc_kernel<256,2,3>(', 'colsum_kernel']


def test_cases_reach_native_plan_classes():
    """every plan class of the native pyramids (every layer, level and B = 1..8) is reached by a GPU case below"""
    fwd_native, fwd_cases, wg_native, wg_cases = set(), set(), set(), set()
    for geo in PYRAMIDS:
        levels = _levels(geo)
        w = PYRAMIDS[geo][1]
        for B in range(1, 9):
            for Cin, Cout in ((w, w), (w, A * K_CLS), (w, A * 4), (A * K_CLS, w), (A * 4, w)):
                fwd_native |= _conv_features(_conv_plan(levels, B, Cin, Cout))
            for Cout in (w, A * K_CLS, A * 4):
                for h, ww in levels:
                    if _box(B, h, ww) is None:
                        wg_native |= _wgrad_features(_wgrad_plan(B, h, ww, w, Cout, SMS))
    for geo in FWD_PYRAMIDS:
        for layer in FWD_LAYERS:
            Cin, Cout = _channels(geo, layer)
            fwd_cases |= _conv_features(_conv_plan(_levels(geo), _fwd_batch(layer), Cin, Cout))
        for layer in DGRAD_LAYERS:
            Cout, Cin = _channels(geo, layer)
            fwd_cases |= _conv_features(_conv_plan(_levels(geo), _dgrad_batch(layer), Cin, Cout))
    cps = []
    for geo, layer, B in WGRAD_CASES:
        Cin, Cout = _channels(geo, layer)
        for h, w in _levels(geo):
            if _box(B, h, w) is None:
                p = _wgrad_plan(B, h, w, Cin, Cout, SMS)
                wg_cases |= _wgrad_features(p)
                cps.append(p['cps'])
    assert fwd_native <= fwd_cases, fwd_native - fwd_cases
    assert wg_native <= wg_cases, wg_native - wg_cases
    # the classes the launchers distinguish, each reached
    assert {('kblocks', k) for k in (1, 2, 3, 5, 6, 12)} | {('tile', 128, 6), ('tile', 64, 1), 'level with M < 128'} \
        <= fwd_cases
    assert {'cap', 'min8', 'one split', 'free', ('ctiles', 1), ('ctiles', 2), ('ntiles', 6)} <= wg_cases
    # the K range of one CTA: the cases reach the native pyramids' longest at B = 1 and 2 (58-61 chunks, P3 of d5, d6)
    native_cps = [_wgrad_plan(B, h, w, PYRAMIDS[geo][1], Cout, SMS)['cps'] for geo in PYRAMIDS for B in (1, 2)
                  for Cout in (PYRAMIDS[geo][1], A * K_CLS, A * 4) for h, w in _levels(geo) if _box(B, h, w) is None]
    assert max(native_cps) <= WG_MAX_CHUNKS_PER_SPLIT and max(cps) >= 58 and sorted(cps)[-2] >= 58, (native_cps, cps)
    assert any(_box(B, h, w) is not None for geo, _, B in WGRAD_CASES for h, w in _levels(geo))


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device=_dev())


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _buffer(levels, B, C, head):
    """a NaN-filled fp32 buffer holding every level, followed by GUARD NaN elements: the concatenated [B, sum(HWA), C/A]
    layout of RetinaHeadFn (head) or dense [B, H, W, C] maps one after the other.  -> (buffer, number of elements in use,
    per level (pointer, batch stride in elements, [B, H, W, C] view))"""
    if head:
        width = C // A
        offs, tot = [], 0
        for h, w in levels:
            offs.append(tot)
            tot += h * w * A
        n = B * tot * width
        buf = torch.full((n + GUARD,), float('nan'), device=_dev())
        v = buf[:n].view(B, tot, width)
        lv = [(buf.data_ptr() + 4 * off * width, tot * width, v[:, off:off + h * w * A].view(B, h, w, C))
              for off, (h, w) in zip(offs, levels)]
    else:
        n = sum(B * h * w * C for h, w in levels)
        buf = torch.full((n + GUARD,), float('nan'), device=_dev())
        lv, off = [], 0
        for h, w in levels:
            lv.append((buf.data_ptr() + 4 * off, h * w * C, buf[off:off + B * h * w * C].view(B, h, w, C)))
            off += B * h * w * C
    return buf, n, lv


def _check_written(buf, n, what):
    assert not torch.isnan(buf[:n]).any(), ('%s: an output element was not written' % what)
    assert torch.isnan(buf[n:]).all(), ('%s: written past the end of the output' % what)


def _check_launch(launch, plan, what):
    name = 'conv_tc_kernel<%d,%d,3>(' % (plan['BN'], plan['stages'])
    print('  %s: %s grid %s' % (what, name, launch))
    assert len(launch) == 1 and launch[0][1] == plan['grid'] and name in launch[0][0], (launch, plan)


def _level_ctrl(got, want):
    """control: the worst level against a reference without the smallest level"""
    return max(_rel(g, w) for g, w in zip(got, want[:-1] + [torch.zeros_like(want[-1])]))


def _rel(got, want):
    """||got - want|| / ||want|| on the device; against a zero reference 1 (or 0 when got is zero too)"""
    n = float(want.norm())
    return float((got.double() - want).norm()) / n if n > 0 else float(float(got.norm()) > 0)


def _weights(g, Cout, Cin):
    return _randn(g, Cout, Cin, 3, 3) * (1.0 / (9 * Cin) ** 0.5), _randn(g, Cout) * 0.1


# ------------------------------------------------------------------------------------------------
# the calls of the GPU tests, and their launches recorded in a process of their own
# ------------------------------------------------------------------------------------------------

def _fwd_setup(ops, geo, layer):
    """inputs of a forward case and launch(act) -> (output buffer, elements in use, per-level [B, H, W, Cout] views)"""
    levels = _levels(geo)
    Cin, Cout = _channels(geo, layer)
    B = _fwd_batch(layer)
    g = _gen(Cin * 1000 + Cout + B)
    xs = [_randn(g, B, h, w, Cin) for h, w in levels]
    w, bias = _weights(g, Cout, Cin)
    wf, _ = ops.pack_conv(w)
    fwd, _ = ops.tc_packs(w)

    def launch(a):
        buf, n, lv = _buffer(levels, B, Cout, _head(layer))
        ops.conv2d_multi_raw(xs[0], [dict(x_ptr=x.data_ptr(), x_bs=h * w_ * Cin, y_ptr=p, y_bs=bs, B=B, H=h, W=w_)
                                     for x, (h, w_), (p, bs, _) in zip(xs, levels, lv)], wf, Cin, Cout, 3, bias=bias, act=a,
                             w_tc=fwd)
        return buf, n, [v for _, _, v in lv]
    act = {'relu': ops.ACT_RELU, 'none': ops.ACT_NONE, 'sigmoid': ops.ACT_SIGMOID}[FWD_LAYERS[layer]]
    return dict(levels=levels, Cin=Cin, Cout=Cout, B=B, xs=xs, w=w, bias=bias, act=act, launch=launch)


def _dgrad_setup(ops, geo, layer):
    """inputs of a data-gradient case (the gradient written into the concatenated head buffer for the class and box
    convs) and launch() -> (output buffer, elements in use, per-level [B, H, W, Cin] views)"""
    levels = _levels(geo)
    Cin, Cout = _channels(geo, layer)                 # of the forward layer: the gradient runs Cout -> Cin
    B = _dgrad_batch(layer)
    g = _gen(Cout * 1000 + Cin + B + 7)
    w, _ = _weights(g, Cout, Cin)
    _, wd = ops.pack_conv(w)
    _, dgr = ops.tc_packs(w)
    src, _, slv = _buffer(levels, B, Cout, _head(layer))
    dys = []
    for (h, w_), (_, _, v) in zip(levels, slv):
        v.copy_(_randn(g, B, h, w_, Cout))
        dys.append(v)
    extra = [_randn(g, B, h, w_, Cin) for h, w_ in levels]      # the mask source, or the residual of the first layer
    first = layer == 'first'

    def launch():
        buf, n, lv = _buffer(levels, B, Cin, False)
        lvs = []
        for (h, w_), (xp, xbs, _), (p, bs, _), e in zip(levels, slv, lv, extra):
            d = dict(x_ptr=xp, x_bs=xbs, y_ptr=p, y_bs=bs, B=B, H=h, W=w_)
            if first:
                d.update(res_ptr=e.data_ptr(), res_bs=h * w_ * Cin)
            else:
                d.update(mask_ptr=e.data_ptr(), mask_bs=h * w_ * Cin)
            lvs.append(d)
        ops.conv2d_multi_raw(extra[0], lvs, wd, Cout, Cin, 3, w_tc=dgr)
        return buf, n, [v for _, _, v in lv]
    return dict(levels=levels, Cin=Cin, Cout=Cout, B=B, w=w, src=src, dys=dys, extra=extra, first=first, launch=launch)


def _wgrad_setup(ops, geo, layer, B):
    """inputs of a weight-gradient case (dy in the concatenated head buffer for the class and box convs) and
    launch(levels, dw, dbias), which adds the gradients of those levels to dw and dbias"""
    levels = _levels(geo)
    Cin, Cout = _channels(geo, layer)
    g = _gen(Cin * 1000 + Cout + B + 13)
    xs = [_randn(g, B, h, w, Cin) for h, w in levels]
    src, _, slv = _buffer(levels, B, Cout, _head(layer))
    dys = []
    for (h, w), (_, _, v) in zip(levels, slv):
        v.copy_(_randn(g, B, h, w, Cout))
        dys.append(v)

    def launch(ls, dw, db):
        lv = [dict(x_ptr=xs[i].data_ptr(), x_bs=levels[i][0] * levels[i][1] * Cin, dy_ptr=slv[i][0], dy_bs=slv[i][1], B=B,
                   H=levels[i][0], W=levels[i][1]) for i in ls]
        ops.conv_wgrad_multi(xs[0], lv, dw, db, Cin, Cout, 3, tc=True)
    return dict(levels=levels, Cin=Cin, Cout=Cout, g=g, xs=xs, src=src, dys=dys, launch=launch)


WGRAD_KERNELS = ('wgrad_tc_kernel', 'colsum_kernel', 'wgrad_tc2_multi_kernel')


def _record_launches(out_dir):
    """run every call of the GPU tests once under torch.profiler; write {case: [(kernel name, grid)]} to
    out_dir/launches.json"""
    from models import _ops as ops
    ops.PRECISION = 'bf16x3'
    out_dir = pathlib.Path(out_dir)
    rec = {}
    for geo in FWD_PYRAMIDS:
        for layer in FWD_LAYERS:
            s = _fwd_setup(ops, geo, layer)
            rec['fwd %s %s' % (geo, layer)] = _launches(lambda: s['launch'](s['act']), out_dir, 'conv_tc_kernel')
        for layer in DGRAD_LAYERS:
            s = _dgrad_setup(ops, geo, layer)
            rec['dgrad %s %s' % (geo, layer)] = _launches(s['launch'], out_dir, 'conv_tc_kernel')
    for geo, layer, B in WGRAD_CASES:
        s = _wgrad_setup(ops, geo, layer, B)
        dw = torch.zeros(s['Cout'], s['Cin'], 3, 3, device=_dev())
        db = torch.zeros(s['Cout'], device=_dev())
        n = len(s['levels'])
        for key, ls in [(str(i), [i]) for i in range(n)] + [('all', list(range(n)))]:
            trace = _launches(lambda: s['launch'](ls, dw, db), out_dir, '_kernel')
            rec['wgrad %s %s %d %s' % (geo, layer, B, key)] = [t for t in trace if any(k in t[0] for k in WGRAD_KERNELS)]
        del s
    with open(out_dir / 'launches.json', 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def launches(tmp_path_factory):
    """the kernel names and grids of every call below, recorded by _record_launches in a fresh interpreter: a CUDA
    activity trace in a long test process can miss this library's kernels after some of the other tests have run"""
    out = tmp_path_factory.mktemp('gather_launches')
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    path = [here, os.path.join(repo, 'oracle'), os.path.join(repo, 'efficientdet.pytorch_b200'), repo]
    code = 'import sys; sys.path[:0] = %r; import test_gather_path_parity as T; T._record_launches(%r)' % (path, str(out))
    subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], check=True, cwd=repo,
                   timeout=1200)
    with open(out / 'launches.json') as f:
        return {k: [(name, tuple(grid)) for name, grid in v] for k, v in json.load(f).items()}


# ------------------------------------------------------------------------------------------------
# 1. forward: conv_tc_kernel over five levels in one launch
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('layer', list(FWD_LAYERS))
@pytest.mark.parametrize('geo', FWD_PYRAMIDS)
def test_forward_one_launch(ops, geo, layer, launches):
    """the layer on all five levels in one launch, with its bias and activation, into the layout RetinaHeadFn writes
    (class and box convs: level slices of one concatenated output, batch stride sum(HWA) * width); NaN guard after the
    output; controls: a reference without the smallest level, one bf16 product per multiply-add (without activation)"""
    s = _fwd_setup(ops, geo, layer)
    levels, Cin, Cout, B, xs, w, bias = (s[k] for k in ('levels', 'Cin', 'Cout', 'B', 'xs', 'w', 'bias'))
    buf, n, got = s['launch'](s['act'])
    lin = [_nhwc(F.conv2d(_nchw(x), w.double(), bias.double(), 1, 1)) for x in xs]
    f = {'relu': torch.relu, 'none': lambda t: t, 'sigmoid': torch.sigmoid}[FWD_LAYERS[layer]]
    want = [f(t) for t in lin]
    what = '%s %s %d->%d %s B=%d' % (layer, FWD_LAYERS[layer], Cin, Cout, geo, B)
    _check(got, want, what)
    _check_written(buf, n, what)
    plan = _conv_plan(levels, B, Cin, Cout)
    _check_launch(launches['fwd %s %s' % (geo, layer)], plan, '%d K blocks, tiles begin %s' % (plan['kblocks'],
                                                                                                plan['tile_begin']))
    miss = _level_ctrl(got, want)
    with _single_pass(ops):
        _, _, single = s['launch'](ops.ACT_NONE)
    single = _rel(torch.cat([t.flatten() for t in single]), torch.cat([t.flatten() for t in lin]))
    print('  controls: without the smallest level %.2e, single pass %.2e' % (miss, single))
    assert miss > TOL_LOCAL and single > SINGLE_PASS_MIN, (miss, single)


# ------------------------------------------------------------------------------------------------
# 2. data gradient: conv_tc_kernel on the dgrad pack
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('layer', DGRAD_LAYERS)
@pytest.mark.parametrize('geo', FWD_PYRAMIDS)
def test_data_gradient_one_launch(ops, geo, layer, launches):
    """dx of the layer Cin -> Cout as RetinaHeadFn.backward launches it: class and box convs read their gradient from the
    concatenated [B, sum(HWA), width] buffer (x batch stride sum(HWA) * width) and apply the ReLU mask of the tower
    output; the tower layers apply the mask, the first tower layer adds a residual.  Masks come from separate random
    tensors, so none can flip.  Controls: a reference without the smallest level, one bf16 product per multiply-add"""
    s = _dgrad_setup(ops, geo, layer)
    levels, Cin, Cout, B, w, dys, extra, first = (s[k] for k in ('levels', 'Cin', 'Cout', 'B', 'w', 'dys', 'extra',
                                                                 'first'))
    buf, n, got = s['launch']()
    tr = [_nhwc(F.conv_transpose2d(_nchw(d), w.double(), None, 1, 1)) for d in dys]
    want = [t + e.double() for t, e in zip(tr, extra)] if first else [t * (e > 0) for t, e in zip(tr, extra)]
    what = '%s data gradient %d->%d %s B=%d%s' % (layer, Cout, Cin, geo, B, ' + residual' if first else ', ReLU mask')
    _check(got, want, what)
    _check_written(buf, n, what)
    plan = _conv_plan(levels, B, Cout, Cin)
    _check_launch(launches['dgrad %s %s' % (geo, layer)], plan, '%d K blocks, tiles begin %s' % (plan['kblocks'],
                                                                                                  plan['tile_begin']))
    miss = _level_ctrl(got, want)
    with _single_pass(ops):
        _, _, single = s['launch']()
    # against the convolution alone: the residual would dilute the single-pass error
    if first:
        single = [t.double() - e.double() for t, e in zip(single, extra)]
        want = tr
    single = _rel(torch.cat([t.flatten() for t in single]), torch.cat([t.flatten() for t in want]))
    print('  controls: without the smallest level %.2e, single pass %.2e' % (miss, single))
    assert miss > TOL_LOCAL and single > SINGLE_PASS_MIN, (miss, single)


# ------------------------------------------------------------------------------------------------
# 3. weight gradient: wgrad_tc_kernel + colsum_kernel, and wgrad_tc2_multi_kernel on the boxed levels of D2 and D7
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('geo,layer,B', WGRAD_CASES)
def test_weight_gradient(ops, geo, layer, B, launches):
    """conv_wgrad_multi as RetinaHeadFn.backward calls it (tc=True, workspaces, dbias; the class and box convs read dy
    from the concatenated buffer), each level alone and then all levels in one call, accumulated into a non-zero dw and
    dbias.  Controls: the dw reference without the first 64 chunks (4 096 pixels) of P3, the dbias reference without the
    last level, one bf16 product per multiply-add"""
    s = _wgrad_setup(ops, geo, layer, B)
    levels, Cin, Cout, g, xs, dys = (s[k] for k in ('levels', 'Cin', 'Cout', 'g', 'xs', 'dys'))
    shape = (Cout, Cin, 3, 3)
    refs = [torch.nn.grad.conv2d_weight(_nchw(x), shape, _nchw(d), 1, 1) for x, d in zip(xs, dys)]
    sums = [d.double().sum(dim=(0, 1, 2)) for d in dys]
    total, total_b = sum(refs), sum(sums)
    dw0 = _randn(g, *shape) * float(total.std())
    db0 = _randn(g, Cout) * float(total_b.pow(2).mean().sqrt())

    def launch(ls):
        dw, db = dw0.clone(), db0.clone()
        s['launch'](ls, dw, db)
        return dw.double() - dw0.double(), db.double() - db0.double()

    def check_launches(key, ls):
        got = launches['wgrad %s %s %d %s' % (geo, layer, B, key)]
        want = _wgrad_launches(B, [levels[i] for i in ls], Cin, Cout, sms)
        assert len(got) == len(want) and all(nm in g_[0] and (grid is None or grid == g_[1])
                                             for (nm, grid), g_ in zip(want, got)), (got, want)
        return got

    def check_db(got, want, what):
        e = _rel(got, want)
        print('  %s dbias rel err %.2e (bound %.0e)' % (what, e, TOL_SUM))
        assert e < TOL_SUM, (what, e)

    sms = _sms()
    what = '%s wgrad %d->%d %s B=%d' % (layer, Cin, Cout, geo, B)
    for i, (h, w) in enumerate(levels):
        dw, db = launch([i])
        p = _wgrad_plan(B, h, w, Cin, Cout, sms)
        route = 'TMA' if _box(B, h, w) else '%d chunks per split (%s)' % (p['cps'], p['rule'])
        _check_dw(dw, refs[i], '%s level %dx%d alone, %s' % (what, h, w, route))
        check_db(db, sums[i], 'level %dx%d' % (h, w))
        check_launches(str(i), [i])
    dw, db = launch(range(len(levels)))
    _check_dw(dw, total, '%s all levels' % what)
    check_db(db, total_b, 'all levels')
    print('  launches: %s' % check_launches('all', range(len(levels))))
    # controls
    h, w = levels[0]
    d_first = torch.zeros(1, h * w, Cout, device=_dev())
    d_first[:, :64 * WG_MAX_CHUNKS_PER_SPLIT] = dys[0][:1].reshape(1, h * w, Cout)[:, :64 * WG_MAX_CHUNKS_PER_SPLIT]
    first = torch.nn.grad.conv2d_weight(_nchw(xs[0][:1]), shape, _nchw(d_first.view(1, h, w, Cout)), 1, 1)
    miss_chunks = max(_block_errs(dw, total - first))
    miss_level = _rel(db, total_b - sums[-1])
    with _single_pass(ops):
        single = _rel(launch(range(len(levels)))[0], total)
    print('  controls: dw without the first 64 chunks of P3 worst block %.2e, dbias without the last level %.2e, '
          'single pass %.2e' % (miss_chunks, miss_level, single))
    assert miss_chunks > TOL_LOCAL and miss_level > TOL_SUM and single > SINGLE_PASS_MIN, (miss_chunks, miss_level, single)
