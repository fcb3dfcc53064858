"""Kernel-level fp64 parity of the single-pass (bf16 mode) tensor-core instances at the launch plans that mode runs.

With EFFDET_B200_PRECISION=bf16 every dense 3x3 conv of neck and head takes one bf16 product per multiply-add: the
NP = 1 instances of the tensor-core kernels (template argument NP, the tc_single flag of the C ABI).  Their producers
store hi8 instead of split8, their TMA producers expect other transaction byte counts and skip the lo loads, and
wg_mma / wg_mma_mn_steps take another branch, so they are code of their own.  This file

  * records, with tests/test_host_trace.py's Recorder (nothing is computed), the bf16-mode calls of bench.py's d0 train
    step (512^2, B = 32) and d4 train step (1024^2, B = 4), of the d7 1536^2 B = 1 forward tools/bench_precision.py
    times, and of a D2 768^2 and a D7 1536^2 train step at B = 1, where one weight-gradient call mixes
    wgrad_tc2_multi_kernel levels with wgrad_tc_kernel levels; every 3x3 call must carry tc_single = 1 and every 1x1
    call tc_single = 0;
  * sorts every recorded call into plan classes with the launcher mirrors of tests/test_planes_path_parity.py and
    tests/test_gather_path_parity.py, each class named by its NP = 1 instance, and checks that the GPU cases (CASES),
    every one a recorded call, reach every class of the traces and their longest accumulations (the most pixel chunks
    one weight-gradient CTA accumulates, the most K blocks per tap, the most persistent units of one conv_planes CTA),
    and that removing any one case loses a class;
  * runs every case once under torch.profiler in an interpreter of its own: kernel names must be the NP = 1 instances
    and grids must match the mirrors;
  * holds every case, into NaN-filled outputs followed by a NaN guard, to a float64 reference on the device built from
    the bf16 values the kernel multiplies: the hi plane's bits of operands handed over as planes, rn(t) (round to
    nearest even, as __float2bfloat16_rn) of fp32 operands the kernel gathers and rounds itself and of the weights.
    Bias, activation, residual, ReLU mask, column sums and dbias are applied in float64 to the unrounded values, as the
    kernels apply them in fp32;
  * runs a differential check that needs no reference: on operands that are already bf16-exact (every lo plane zero)
    the bf16 and the bf16x3 instance add the same products and exact zeros into the same fp32 accumulators, so
    outputs, output planes and ReLU-mask bits must be bit-identical, and so must a weight gradient whose every launch
    runs in one split.  Weight gradients over several splits and column sums add with fp32 atomics in no fixed
    order; there bf16 vs bf16x3 is held to the larger of twice the difference between two bf16x3 runs and 1e-6.

Bounds (norm-relative error, as tests/test_planes_path_parity.py):
  TOL_TC    = 3e-5  each whole call
  TOL_LOCAL = 1e-4  each pyramid level of a forward or data-gradient output, each 64-output-channel x tap block of dw
  TOL_SUM   = 2e-5  dbias and column sums
Products of bf16 values are exact in fp32, so what is left is the fp32 accumulation, as in bf16x3.
Controls, each of which must fail its bound: the same call in bf16x3 against the rounded reference (the reference
tells one product from three), the single-pass result against the unrounded reference (above SINGLE_PASS_MIN), and a
structural one: the reference without the smallest level, or for a weight gradient without the first 64 chunks
(4 096 pixels) of P3.

wgrad_tc_kernel<64,4,1> is reached by no traced configuration: it serves levels without a pixel box at Cin <= 64, and
only D0 has such widths, where every level has a box.  Its coverage stays with tests/test_bf16_mode.py
(test_gathering_kernels_single_pass, 64 -> 64 on a 2x2 map).

Measured on an H100 80GB HBM3 at 700 W (132 SMs), the worst case of each instance (whole call / worst level or block):
  conv_planes_kernel<128,1>          7.49e-6 / 7.50e-6   d4 class conv data gradient 720 -> 256, 12 K blocks
  conv_planes_kernel<64,1>           2.36e-6 / 2.36e-6   d4 box conv 256 -> 36
  conv_tc_kernel<128,3,1>            7.05e-6 / 7.07e-6   D2 class conv data gradient 720 -> 256
  conv_tc_kernel<64,4,1>             2.35e-6 / 2.36e-6   D2 box conv 256 -> 36
  wgrad_tc2_multi_kernel<256,2,1>    4.32e-6 / 4.39e-6   d0 box conv, 64 chunks per CTA (the cap binds)
  wgrad_tc2_multi_kernel<64,4,1>     4.34e-6 / 4.42e-6   d0 BiFPN node on 64x64, 64 chunks per CTA
  wgrad_tc_kernel<256,2,1>           1.86e-6 / 1.89e-6   D7 BiFPN node on 96x96, 29 chunks per CTA
  column sums 7.48e-6, dbias 7.83e-7
All at or below the bf16x3 figures of the same plans (1.2-2.3e-5): the products are exact, and the error grows with the
reduction length as there.  The weakest controls: one product per multiply-add against the unrounded reference
9.06e-4 (the sigmoid class conv at d0; 2.3e-3 elsewhere), bf16x3 against the rounded reference the same, column sums
without the smallest level 5.03e-2, dbias without the last level 3.96e-2, dw without the first 64 chunks of P3 0.160
(worst block).  The differential check was bit-exact for every forward and data gradient (outputs, output planes, ReLU
bits) and for the single-split weight gradient.  Over several splits bf16 vs bf16x3 differed by at most 1.45e-7, within
twice what two bf16x3 runs differed by, except on the D7 96x96 level (5.0e-8 against 7.2e-9), which the 1e-6 floor
covers: the atomics order of a few splits is often the same twice.  Column sums 2.2e-7 against 2.0e-7.  No kernel
disagreed.  The file's GPU
tests take about 50 s there."""
import collections
import json
import os
import pathlib
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O
from test_benchmark_plans import _launches
from test_gather_path_parity import (GUARD, NO_BOX, PYRAMIDS, _buffer, _check_written, _conv_plan, _rel,
                                     _wgrad_launches, _wgrad_plan)
from test_host_trace import Recorder
from test_planes_path_parity import (SINGLE_PASS_MIN, TOL_LOCAL, TOL_SUM, TOL_TC, WG_MAX_CHUNKS_PER_SPLIT, _block_errs,
                                     _box, _check, _check_dw, _chunks, _split_plan)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(REPO, 'tools') not in sys.path:
    sys.path.insert(0, os.path.join(REPO, 'tools'))
from bf16_emulation import rn  # noqa: E402

SMS = 132                       # H100 SXM: the SM count the plans are walked at
A = 9                           # anchors per pixel
ACTS = {0: 'none', 1: 'relu', 3: 'sigmoid'}
DIFF_FLOOR = 1e-6               # least bound of the atomics-order difference between bf16 and bf16x3


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------
# the recorded traces
# ------------------------------------------------------------------------------------------------

# name: (network, classes, W_bifpn, D_bifpn, input size, batch, train); d0, d4 are bench.CONFIGS' train configs, d7i the
# forward tools/bench_precision.py times (bench.CONFIGS['d7']), d2 and d7 train steps of those pyramids
TRACES = {'d0': ('efficientdet-d0', 80, 64, 2, 512, 32, True), 'd4': ('efficientdet-d4', 80, 224, 6, 1024, 4, True),
          'd7i': ('efficientdet-d7', 80, 384, 8, 1536, 1, False), 'd2': ('efficientdet-d2', 80, 112, 5, 768, 1, True),
          'd7': ('efficientdet-d7', 80, 384, 8, 1536, 1, True)}
CONV_CALLS = {'effdet_conv2d': 'conv', 'effdet_conv2d_multi': 'conv', 'effdet_conv2d_wgrad': 'wgrad',
              'effdet_conv2d_wgrad_multi': 'wgrad', 'effdet_conv_planes_multi': 'planes'}


def _record_traces():
    """{trace: [(call kind, fwd | dgrad | wgrad, [level argument dicts])]} of the 1x1 and 3x3 conv calls of one bf16-mode
    step (the second, steady-state one of a train step)"""
    import __graft_entry__ as entry
    entry.build()
    from bench import CONFIGS
    from models import EfficientDet, _native as N, _ops
    for name in ('d0', 'd4', 'd7'):
        c = CONFIGS[name]
        t = TRACES[name if name != 'd7' else 'd7i']
        assert t == (c['net'], c['K'], c['W'], c['D'], c['size'], c['bs'], c['mode'] == 'train'), name
    assert all(TRACES[g][2] == PYRAMIDS[p][1] and TRACES[g][4] == PYRAMIDS[p][0]
               for g, p in (('d2', 'd2_768'), ('d7', 'd7_1536')))
    rec = Recorder()
    traces = {}
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(N, 'f32', rec.f32)
        mp.setattr(N, 'ptr', rec.ptr)
        mp.setattr(N, 'call', rec.call)
        mp.setattr(_ops, 'check_cuda_f32', lambda x, what: None)
        mp.setattr(_ops, '_cache', {})
        mp.setattr(_ops, 'PRECISION', 'bf16')
        for name, (net, K, W, D, size, B, train) in TRACES.items():
            cfg = O.make_config(net, K, W, D)
            m = EfficientDet(num_classes=K, network=net, D_bifpn=D, W_bifpn=W, is_training=True)
            m.load_state_dict(O.init_state_dict(cfg, seed=0))
            images, ann = O.synthetic_batch(B, size=size, num_classes=K, seed=3)
            if train:
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
            traces[name] = [(CONV_CALLS[n], 'wgrad' if CONV_CALLS[n] == 'wgrad' else 'fwd' if i < back else 'dgrad',
                             s[0] if isinstance(s[0], list) else [s[0]])
                            for i, (n, s) in enumerate(rec.calls) if i >= start and n in CONV_CALLS]
            del m, images, ann
    return traces


# ------------------------------------------------------------------------------------------------
# signatures: what a GPU case needs to repeat one recorded 3x3 call
# ------------------------------------------------------------------------------------------------

def _signature(call, kind, levels):
    """planes: (planes, fwd | dgrad, Cin, Cout, B, ((H, W) per level), act, epilogue) with epilogue the tuple of bias,
    y (fp32 output), y strided (a concatenated head buffer), y_planes, y_mask, mask_planes, mask_bits, residual,
    colsum that the call passes;
    conv: (conv, fwd | dgrad, Cin, Cout, B, levels, act, epilogue) with bias, x strided, y strided, residual, mask_src;
    wgrad: (wgrad, wgrad, Cin, Cout, B, levels, 'none', operands) with planes or fp32, dy strided, dbias"""
    a = levels[0]
    B, Cin, Cout = a['B'], a['Cin'], a['Cout']
    hw = tuple((lv['H'], lv['W']) for lv in levels)

    def strided(f, C):
        return any(lv[f + '_bstride'] != lv['H'] * lv['W'] * C for lv in levels if lv[f] is not None)
    if call == 'planes':
        epi = tuple(f for f in ('bias', 'y') if a[f] is not None)
        epi += ('y strided',) if strided('y', Cout) else ()
        epi += tuple(f for f in ('y_planes', 'y_mask', 'mask_planes', 'mask_bits', 'residual', 'colsum') if a[f] is not None)
        return ('planes', kind, Cin, Cout, B, hw, ACTS[a['act']], epi)
    if call == 'conv':
        epi = ('bias',) if a['bias'] is not None else ()
        epi += ('x strided',) if strided('x', Cin) else ()
        epi += ('y strided',) if strided('y', Cout) else ()
        epi += tuple(f for f in ('residual', 'mask_src') if a[f] is not None)
        return ('conv', kind, Cin, Cout, B, hw, ACTS[a['act']], epi)
    ops = ('planes',) if a['x_planes'] is not None else ('fp32',)
    assert (a['x_planes'] is None) == (a['dy_planes'] is None), a
    ops += ('dy strided',) if strided('dy', Cout) else ()
    ops += ('dbias',) if a['dbias'] is not None else ()
    return ('wgrad', 'wgrad', Cin, Cout, B, hw, 'none', ops)


# ------------------------------------------------------------------------------------------------
# mirrors of the launchers, extended by the NP = 1 instance suffix, and the plan classes
# ------------------------------------------------------------------------------------------------

def _kstage(B, h, w):
    """pixels of one pixel box (wg_geometry, conv_tc.cu)"""
    Wb = w if w <= 64 else 64
    Hb = max(t for t in range(1, h + 1) if h % t == 0 and Wb * t <= 64)
    return Wb * Hb * _box(B, h, w)[0]


def _planes_plan(B, hw, Cin, Cout, sms=SMS):
    """effdet_conv_planes_multi (conv_planes.cu): tile width, 128-row tiles of all levels, channel tiles, persistent grid,
    units of the busiest CTA"""
    BN = 64 if Cout <= 64 else 128
    tiles = sum(_cdiv(_chunks(B, h, w), 128 // _kstage(B, h, w)) for h, w in hw)
    units = tiles * _cdiv(Cout, BN)
    grid = min(units, sms)
    return dict(BN=BN, kernel='conv_planes_kernel<%d,1>(' % BN, tiles=tiles, ntn=_cdiv(Cout, BN), kblocks=_cdiv(Cin, 64),
                partial=Cout % BN != 0, grid=(grid, 1, 1), busiest=_cdiv(units, grid))


def _units_class(n):
    """persistent units of the busiest CTA: one warpgroup only, one hand-over, then odd and even counts (the k-th unit
    belongs to consumer warpgroup k & 1)"""
    return n if n <= 2 else 'odd > 2' if n % 2 else 'even > 2'


def _single(name):
    return name.replace(',3>(', ',1>(')


def _wgrad_route(B, hw, Cin, Cout, sms=SMS):
    """[(kernel name, grid or None, plan)] of one weight-gradient call (conv2d_wgrad in conv_api.cu): all levels in one
    wgrad_tc2_multi_kernel launch when every level has a pixel box and there are several, else one route per level"""
    if len(hw) > 1 and all(_box(B, h, w) is not None for h, w in hw):
        begins, n, cps, splits = _split_plan(B, list(hw), Cin, Cout, sms)
        BC = 256 if Cin > 64 else 64
        return [('wgrad_tc2_multi_kernel<%d,%d,1>(' % (BC, 2 if BC == 256 else 4),
                 (_cdiv(Cin, BC) * _cdiv(Cout, 128), 9, splits), dict(levels=list(hw)))]
    out = []
    for (name, grid), lv in zip([t for t in _wgrad_launches(B, list(hw), Cin, Cout, sms) if t[0] != 'colsum_kernel'], hw):
        out.append((_single(name), grid, dict(levels=[lv])))
        if name.startswith('wgrad_tc_kernel'):
            out.append(('colsum_kernel', None, None))
    return out


def _tc2_features(B, levels, Cin, Cout, sms=SMS):
    """split-K placement of one wgrad_tc2_multi_kernel launch: the cap binds, one split, one chunk per split, a split
    boundary inside a level (and a split that straddles two levels)"""
    begins, n, cps, splits = _split_plan(B, levels, Cin, Cout, sms)
    f = set()
    if _split_plan(B, levels, Cin, Cout, sms, cap=None)[2] > WG_MAX_CHUNKS_PER_SPLIT:
        f.add('cap binds')
    if splits == 1 and cps > 1:
        f.add('one split')
    if cps == 1:
        f.add('one chunk per split')
    if len(levels) > 1:
        ends = begins[1:] + [n]
        inside = any(b0 < k * cps < e for k in range(1, splits) for b0, e in zip(begins, ends))
        straddle = any(s * cps < b0 < (s + 1) * cps for s in range(splits) for b0 in begins[1:])
        if inside and straddle:
            f.add('boundary inside a level')
    return f, cps


def _classes(sig, sms=SMS):
    """-> (plan classes, {figure: value}) of one call; the figures are the longest accumulations"""
    call, kind, Cin, Cout, B, hw, act, epi = sig
    cls, fig = set(), {}
    if call == 'planes':
        p = _planes_plan(B, hw, Cin, Cout, sms)
        k = p['kernel']
        cls |= {(k, 'n-tiles', p['ntn'], 'partial' if p['partial'] else 'full'), (k, 'epilogue', act, epi),
                (k, 'units', _units_class(p['busiest'])), (k, 'kblocks', p['kblocks'])}
        fig = {'planes units': p['busiest'], 'kblocks': p['kblocks']}
    elif call == 'conv':
        p = _conv_plan(list(hw), B, Cin, Cout)
        k = 'conv_tc_kernel<%d,%d,1>(' % (p['BN'], p['stages'])
        cls |= {(k, 'n-tiles', p['ntiles']), (k, 'kblocks', p['kblocks'])}
        if p['small']:
            cls.add((k, 'level with M < 128'))
        fig = {'kblocks': p['kblocks']}
    else:
        for name, _, plan in _wgrad_route(B, hw, Cin, Cout, sms):
            if name.startswith('wgrad_tc2'):
                f, cps = _tc2_features(B, plan['levels'], Cin, Cout, sms)
                cls |= {(name, 'n-tiles', _cdiv(Cout, 128))} | {(name, x) for x in f}
                fig['tc2 chunks per CTA'] = max(fig.get('tc2 chunks per CTA', 0), cps)
            elif name.startswith('wgrad_tc_kernel'):
                (h, w), = plan['levels']
                p = _wgrad_plan(B, h, w, Cin, Cout, sms)
                cls |= {(name, p['rule']), (name, 'c-tiles', p['ctiles']), (name, 'n-tiles', p['ntiles'])}
                fig['tc chunks per CTA'] = max(fig.get('tc chunks per CTA', 0), p['cps'])
    return cls, fig


# ------------------------------------------------------------------------------------------------
# the GPU cases: (trace, signature), every one a call of its trace (test_cases_are_recorded_calls)
# ------------------------------------------------------------------------------------------------

D0 = ((64, 64), (32, 32), (16, 16), (8, 8), (4, 4))
D4 = ((128, 128), (64, 64), (32, 32), (16, 16), (8, 8))
D2 = ((96, 96), (48, 48), (24, 24), (12, 12), (6, 6))
D7 = ((192, 192), (96, 96), (48, 48), (24, 24), (12, 12))

CASES = [
    # the class conv of the benchmarked step: 720 outputs in six 128-column tiles (the last 80 wide), sigmoid into the
    # concatenated head buffer; 62 persistent units in the busiest CTA
    ('d0', ('planes', 'fwd', 256, 720, 32, D0, 'sigmoid', ('bias', 'y', 'y strided'))),
    # the head's first tower layer: bias + ReLU into planes and ReLU bits
    ('d0', ('planes', 'fwd', 64, 256, 32, D0, 'relu', ('bias', 'y_planes', 'y_mask'))),
    # its data gradient with the residual of the other tower, 64-column tile
    ('d0', ('planes', 'dgrad', 256, 64, 32, D0, 'none', ('y', 'residual'))),
    # BiFPN node convs on one level: one unit per CTA, and one hand-over
    ('d0', ('planes', 'fwd', 64, 64, 32, ((4, 4),), 'none', ('bias', 'y'))),
    ('d0', ('planes', 'dgrad', 64, 64, 32, ((32, 32),), 'none', ('y',))),
    # the box conv at d4: 36 outputs on the 64-column tile
    ('d4', ('planes', 'fwd', 256, 36, 4, D4, 'none', ('bias', 'y', 'y strided'))),
    # Cin 224 padded to 256 in K, 224 outputs in two tiles (the last 96 wide)
    ('d4', ('planes', 'fwd', 224, 224, 4, ((8, 8),), 'none', ('bias', 'y'))),
    ('d4', ('planes', 'dgrad', 224, 224, 4, ((64, 64),), 'none', ('y',))),
    ('d4', ('planes', 'dgrad', 256, 224, 4, D4, 'none', ('y', 'residual'))),
    # the class conv's data gradient: 12 K blocks per tap, ReLU bits of the tower output, column sums, planes out
    ('d4', ('planes', 'dgrad', 720, 256, 4, D4, 'none', ('y_planes', 'mask_bits', 'colsum'))),
    # gathering forward and data gradient at D2 (levels under 128 pixels) and at D7
    ('d2', ('conv', 'fwd', 256, 720, 1, D2, 'sigmoid', ('bias', 'y strided'))),
    ('d2', ('conv', 'fwd', 256, 36, 1, D2, 'none', ('bias', 'y strided'))),
    ('d2', ('conv', 'fwd', 112, 112, 1, ((6, 6),), 'none', ('bias',))),
    ('d2', ('conv', 'dgrad', 720, 256, 1, D2, 'none', ('x strided', 'mask_src'))),
    ('d2', ('conv', 'dgrad', 36, 256, 1, D2, 'none', ('x strided', 'mask_src'))),
    ('d7i', ('conv', 'fwd', 384, 384, 1, ((12, 12),), 'none', ('bias',))),
    # weight gradients from planes: the cap of 64 chunks per CTA binds, split boundaries inside levels
    ('d0', ('wgrad', 'wgrad', 256, 36, 32, D0, 'none', ('planes',))),
    ('d0', ('wgrad', 'wgrad', 64, 256, 32, D0, 'none', ('planes',))),
    ('d0', ('wgrad', 'wgrad', 64, 64, 32, ((64, 64),), 'none', ('planes',))),
    # weight gradients from fp32 operands that mix wgrad_tc2_multi_kernel and wgrad_tc_kernel levels in one call
    ('d2', ('wgrad', 'wgrad', 256, 720, 1, D2, 'none', ('fp32', 'dy strided', 'dbias'))),
    ('d2', ('wgrad', 'wgrad', 256, 36, 1, D2, 'none', ('fp32', 'dy strided', 'dbias'))),
    ('d2', ('wgrad', 'wgrad', 112, 256, 1, D2, 'none', ('fp32', 'dbias'))),
    # D7 BiFPN weight gradients: two channel tiles of 256 without a pixel box, three n-tiles with one
    ('d7', ('wgrad', 'wgrad', 384, 384, 1, ((96, 96),), 'none', ('fp32', 'dbias'))),
    ('d7', ('wgrad', 'wgrad', 384, 384, 1, ((12, 12),), 'none', ('fp32', 'dbias'))),
]


def _case_id(case):
    name, (call, kind, Cin, Cout, B, hw) = case[0], case[1][:6]
    return '%s-%s-%s-%d-%d-B%d-%dx%d%s' % (name, call, kind, Cin, Cout, B, hw[0][0], hw[0][1],
                                           '-L%d' % len(hw) if len(hw) > 1 else '')


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def traces():
    return _record_traces()


def _calls3(traces):
    """{trace: {signature: level dicts}} of the recorded 3x3 calls"""
    return {name: {_signature(c, k, lv): lv for c, k, lv in calls if lv[0]['ksize'] == 3} for name, calls in traces.items()}


def test_traces_carry_tc_single(traces):
    """every 3x3 call of every trace runs on the tensor cores with tc_single = 1, every 1x1 call with tc_single = 0; the
    D2 and D7 train steps hand their head's weight gradients over in calls that mix the two weight-gradient kernels"""
    n = collections.Counter()
    for name, calls in traces.items():
        for call, kind, levels in calls:
            for a in levels:
                k = a['ksize']
                tc = a['precision'] == 1 if call == 'wgrad' else a['w_tc'] is not None
                assert tc, (name, call, kind, a['Cin'], a['Cout'], k)
                assert a['tc_single'] == (1 if k == 3 else 0), (name, call, kind, a['Cin'], a['Cout'], k)
                n[(name, k)] += 1
    for name in TRACES:
        assert n[(name, 3)] > 20, (name, n)
        assert n[(name, 1)] > 20 or not TRACES[name][6], (name, n)
    for name, pyr in (('d2', 'd2_768'), ('d7', 'd7_1536')):
        mixed = [s for s in _calls3(traces)[name] if s[0] == 'wgrad' and
                 {n_.split('<')[0] for n_, _, _ in _wgrad_route(s[4], s[5], s[2], s[3])} >=
                 {'wgrad_tc2_multi_kernel', 'wgrad_tc_kernel'}]
        assert mixed, name
        assert NO_BOX[pyr] != 'all'


def test_mirrors():
    """the launchers' arithmetic on the figures that motivated the cases (132 SMs)"""
    # d0 class conv: 62 persistent units in the busiest CTA, six n-tiles (the last 80 wide); its data gradient 12 K blocks
    p = _planes_plan(32, D0, 256, 720)
    assert (p['kernel'], p['ntn'], p['partial'], p['grid'], p['busiest']) == ('conv_planes_kernel<128,1>(', 6, True,
                                                                                (132, 1, 1), 62)
    assert _planes_plan(4, D4, 720, 256)['kblocks'] == 12 and _planes_plan(4, ((8, 8),), 224, 224)['kblocks'] == 4
    assert _planes_plan(32, ((4, 4),), 64, 64)['busiest'] == 1
    # d0 weight gradients from planes: one launch over all levels, the cap binds (2728 chunks, 43 splits of 64)
    (name, grid, _), = _wgrad_route(32, D0, 256, 720)
    assert name == 'wgrad_tc2_multi_kernel<256,2,1>(' and grid == (6, 9, 43)
    f, cps = _tc2_features(32, list(D0), 256, 36)
    assert f == {'cap binds', 'boundary inside a level'} and cps == 64
    # a D2 weight gradient: the unboxed 96x96 and 6x6 levels on wgrad_tc_kernel, the others one at a time on wgrad_tc2
    names = [n_ for n_, _, _ in _wgrad_route(1, D2, 256, 720)]
    assert names == ['wgrad_tc_kernel<256,2,1>(', 'colsum_kernel'] + ['wgrad_tc2_multi_kernel<256,2,1>('] * 3 + \
        ['wgrad_tc_kernel<256,2,1>(', 'colsum_kernel']
    assert _wgrad_plan(1, 96, 96, 256, 720, SMS)['cps'] == 29
    # the gathering forward of the class conv at D2: six n-tiles, four K blocks, the 6x6 level under 128 pixels
    c = _conv_plan(list(D2), 1, 256, 720)
    assert (c['BN'], c['ntiles'], c['kblocks'], c['small']) == (128, 6, 4, True)
    assert _conv_plan(list(D2), 1, 720, 256)['kblocks'] == 12


def test_cases_are_recorded_calls(traces):
    """every case repeats a 3x3 call of its trace"""
    recorded = _calls3(traces)
    ids = [_case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids)
    for name, sig in CASES:
        assert sig in recorded[name], (name, sig)


def test_cases_reach_every_plan_class(traces):
    """CASES reach every plan class of the traces and their longest accumulations, and each case is needed: without it
    a class is lost (or, where noted, the longest accumulation of its kernel)"""
    traced, figs = collections.defaultdict(set), {}
    for name, sigs in _calls3(traces).items():
        for sig in sigs:
            cls, fig = _classes(sig)
            for c in cls:
                traced[c].add(name)
            for k, v in fig.items():
                figs[k] = max(figs.get(k, 0), v)
    case_cls = [_classes(sig) for _, sig in CASES]
    covered = set().union(*(c for c, _ in case_cls))
    print()
    for c in sorted(traced, key=str):
        print('  %-90s %s' % (c, ','.join(sorted(traced[c]))))
    missing = set(traced) - covered
    assert not missing, missing
    case_figs = {k: max(f.get(k, 0) for _, f in case_cls) for k in figs}
    print('longest accumulations: traces %s, cases %s' % (figs, case_figs))
    assert case_figs == figs == {'planes units': 62, 'kblocks': 12, 'tc2 chunks per CTA': 64, 'tc chunks per CTA': 29}
    for i, case in enumerate(CASES):
        rest = case_cls[:i] + case_cls[i + 1:]
        lost = covered - set().union(*(c for c, _ in rest))
        assert lost, ('case %s is not needed' % _case_id(case))
    # no traced configuration reaches wgrad_tc_kernel<64,4,1> (see the module docstring)
    assert not any(c[0].startswith('wgrad_tc_kernel<64') for c in traced)


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _dev():
    return torch.device('cuda:0')


def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


class _mode:
    """ops.PRECISION for the launches inside the block"""

    def __init__(self, ops, mode):
        self.ops, self.mode = ops, mode

    def __enter__(self):
        self.old, self.ops.PRECISION = self.ops.PRECISION, self.mode

    def __exit__(self, *exc):
        self.ops.PRECISION = self.old


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _planes_of(ops, x, C):
    """fp32 [B, H, W, C] on the device -> hi/lo planes [2, B, H, W, pitch]"""
    b, h, w, _ = x.shape
    p = ops._planes(b, h, w, C, x)
    ops.to_planes(x.data_ptr(), h * w * C, p, b, h * w, C, x)
    return p


def _guarded(n, dtype, fill):
    """a buffer of n elements followed by GUARD more, all set to fill -> (buffer, first n)"""
    buf = torch.full((n + GUARD,), fill, device=_dev(), dtype=dtype)
    return buf, buf[:n]


def _mask_words(m, C):
    """ReLU bits of a [B, H, W, C] map as _relu_bits lays them out: bit c % 32 of word c // 32 is set when m > 0"""
    words = _cdiv(C, 32)
    bits = torch.zeros(m.shape[:3] + (words * 32,), dtype=torch.int64, device=m.device)
    bits[..., :C] = (m[..., :C] > 0).long()
    v = (bits.view(m.shape[:3] + (words, 32)) << torch.arange(32, device=m.device)).sum(-1)
    return (((v + 2 ** 31) % 2 ** 32) - 2 ** 31).to(torch.int32)


def _i32(t):
    return t.contiguous().view(torch.int32)


def _i16(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------
# one case: operands, the call (in either precision) and its references
# ------------------------------------------------------------------------------------------------

def _setup(ops, case, exact=False):
    """operands of one case (exact: already bf16, so every lo plane is zero) -> dict with launch(mode) -> outputs and
    reference(rounded) -> the float64 values the outputs must match"""
    name, sig = case
    call, kind, Cin, Cout, B, hw, act, epi = sig
    levels = list(hw)
    g = torch.Generator(device=_dev()).manual_seed(sum(map(ord, _case_id(case))) + 7 * exact)

    def randn(*shape):
        t = torch.randn(*shape, generator=g, device=_dev())
        return rn(t) if exact else t
    act_id = {'none': ops.ACT_NONE, 'relu': ops.ACT_RELU, 'sigmoid': ops.ACT_SIGMOID}[act]
    s = dict(call=call, levels=levels, B=B, Cin=Cin, Cout=Cout, act=act, epi=epi)
    if call == 'wgrad':
        return _wgrad_setup(ops, s, randn)
    # the layer's weight: forward Cin -> Cout; a data gradient runs the layer Cout -> Cin backwards
    w = randn(Cout, Cin, 3, 3) * (1.0 / (9 * Cin) ** 0.5) if kind == 'fwd' else randn(Cin, Cout, 3, 3) * (1.0 / (9 * Cin) ** 0.5)
    w = rn(w) if exact else w
    bias = torch.randn(Cout, generator=g, device=_dev()) * 0.1 if 'bias' in epi else None
    res = [torch.randn(B, h, w_, Cout, generator=g, device=_dev()) for h, w_ in levels] if 'residual' in epi else None
    msrc = [torch.randn(B, h, w_, Cout, generator=g, device=_dev()) for h, w_ in levels] \
        if {'mask_src', 'mask_planes', 'mask_bits'} & set(epi) else None
    fwd_pack, dgr_pack = ops.tc_packs(w)
    wtc = fwd_pack if kind == 'fwd' else dgr_pack
    if call == 'planes':
        xs = [randn(B, h, w_, Cin) for h, w_ in levels]
        xp = [_planes_of(ops, x, Cin) for x in xs]
        ops_x = [p[0][..., :Cin].double() for p in xp]             # the hi plane's bits: what the kernel multiplies
        mp = [_planes_of(ops, m, Cout) for m in msrc] if msrc is not None and 'mask_planes' in epi else None
        mbits = [_mask_words(m, Cout) for m in msrc] if msrc is not None and 'mask_bits' in epi else None
        masks = [p[0][..., :Cout].double() > 0 for p in mp] if mp is not None else \
            [m > 0 for m in msrc] if msrc is not None else None
    else:
        src, _, slv = _buffer(levels, B, Cin, 'x strided' in epi)
        xs = []
        for (h, w_), (_, _, v) in zip(levels, slv):
            v.copy_(randn(B, h, w_, Cin))
            xs.append(v)
        ops_x = [rn(x).double() for x in xs]                        # rounded in the kernel's gather
        masks = [m > 0 for m in msrc] if msrc is not None else None
        wf, wd = ops.pack_conv(w)
    s.update(xs=xs, w=w, bias=bias, res=res, masks=masks)

    def launch(mode):
        """-> dict(levels=[B, H, W, Cout] float64 values per level, bits=[tensors that must be bit-identical across modes],
        colsum=..., buffers=[(buffer, n in use)] for the NaN guard, y_mask=...)"""
        out = dict(buffers=[], bits=[])
        with _mode(ops, mode):
            if call == 'planes':
                lvs = [dict(x=xp[i], B=B, H=h, W=w_) for i, (h, w_) in enumerate(levels)]
                if 'y' in epi:
                    buf, n, ylv = _buffer(levels, B, Cout, 'y strided' in epi)
                    for d, (p, bs, _) in zip(lvs, ylv):
                        d.update(y_ptr=p, y_bs=bs)
                    out['buffers'].append((buf, n))
                if 'y_planes' in epi:
                    pitch = ops._pitch8(Cout)
                    yp = []
                    for d, (h, w_) in zip(lvs, levels):
                        n = 2 * B * h * w_ * pitch
                        buf, v = _guarded(n, torch.bfloat16, float('nan'))
                        d['y_planes'] = v.view(2, B, h, w_, pitch)
                        yp.append(d['y_planes'])
                        out['buffers'].append((buf, n))
                if 'y_mask' in epi:
                    ym = []
                    for d, (h, w_) in zip(lvs, levels):
                        n = B * h * w_ * _cdiv(Cout, 32)
                        buf, v = _guarded(n, torch.int32, 0x5a5a5a5a)
                        d['y_mask'] = v.view(B, h, w_, _cdiv(Cout, 32))
                        ym.append((buf, n, d['y_mask']))
                if mp is not None:
                    for d, p in zip(lvs, mp):
                        d['mask'] = p
                if mbits is not None:
                    for d, mb in zip(lvs, mbits):
                        d['mask_bits'] = mb
                if res is not None:
                    for d, r, (h, w_) in zip(lvs, res, levels):
                        d.update(res_ptr=r.data_ptr(), res_bs=h * w_ * Cout)
                colsum = None
                if 'colsum' in epi:
                    start = torch.randn(Cout, generator=torch.Generator(device=_dev()).manual_seed(5), device=_dev())
                    colsum = start.clone()
                ops.conv_planes_multi(xs[0], lvs, wtc, Cin, Cout, 3, bias=bias, act=act_id, colsum=colsum)
                torch.cuda.synchronize()
                if 'y' in epi:
                    out['levels'] = [v.double() for _, _, v in ylv]
                    out['bits'].append(_i32(buf[:n]))
                else:
                    out['levels'] = [(p[0].double() + p[1].double())[..., :Cout] for p in yp]
                    out['bits'] += [_i16(p[..., :Cout]) for p in yp]
                if 'y_mask' in epi:
                    out['y_mask'] = ym
                    out['bits'] += [m for _, _, m in ym]
                if colsum is not None:
                    out['colsum'] = colsum.double() - start.double()
            else:
                buf, n, ylv = _buffer(levels, B, Cout, 'y strided' in epi)
                lvs = []
                for i, ((h, w_), (p, bs, _)) in enumerate(zip(levels, ylv)):
                    d = dict(x_ptr=slv[i][0], x_bs=slv[i][1], y_ptr=p, y_bs=bs, B=B, H=h, W=w_)
                    if res is not None:
                        d.update(res_ptr=res[i].data_ptr(), res_bs=h * w_ * Cout)
                    if msrc is not None:
                        d.update(mask_ptr=msrc[i].data_ptr(), mask_bs=h * w_ * Cout)
                    lvs.append(d)
                ops.conv2d_multi_raw(src, lvs, wf if kind == 'fwd' else wd, Cin, Cout, 3, bias=bias, act=act_id, w_tc=wtc)
                torch.cuda.synchronize()
                out['buffers'].append((buf, n))
                out['levels'] = [v.double() for _, _, v in ylv]
                out['bits'].append(_i32(buf[:n]))
        return out

    def reference(rounded, with_act=True):
        """float64 per level; rounded: from the bf16 operands the kernel multiplies, else from the fp32 operands"""
        wr = (rn(w) if rounded else w).double()
        out = []
        for i, x in enumerate(xs):
            xr = ops_x[i] if rounded else x.double()
            if kind == 'fwd':
                t = _nhwc(F.conv2d(_nchw(xr), wr, None, 1, 1))
            else:
                t = _nhwc(F.conv_transpose2d(_nchw(xr), wr, None, 1, 1))
            if bias is not None:
                t = t + bias.double()
            if with_act:
                t = torch.relu(t) if act == 'relu' else torch.sigmoid(t) if act == 'sigmoid' else t
            if res is not None:
                t = t + res[i].double()
            if masks is not None:
                t = t * masks[i]
            out.append(t)
        return out
    s.update(launch=launch, reference=reference)
    return s


def _wgrad_setup(ops, s, randn):
    levels, B, Cin, Cout, epi = s['levels'], s['B'], s['Cin'], s['Cout'], s['epi']
    planes = 'planes' in epi
    xs = [randn(B, h, w, Cin) for h, w in levels]
    src, _, slv = _buffer(levels, B, Cout, 'dy strided' in epi)
    dys = []
    for (h, w), (_, _, v) in zip(levels, slv):
        v.copy_(randn(B, h, w, Cout))
        dys.append(v)
    if planes:
        xp = [_planes_of(ops, x, Cin) for x in xs]
        dyp = [_planes_of(ops, d.contiguous(), Cout) for d in dys]
        ops_x = [p[0][..., :Cin].double() for p in xp]
        ops_dy = [p[0][..., :Cout].double() for p in dyp]
    else:
        ops_x = [rn(x).double() for x in xs]
        ops_dy = [rn(d).double() for d in dys]
    shape = (Cout, Cin, 3, 3)
    wd = torch.empty(shape, device=_dev())                         # only the device of the launch
    dbias = 'dbias' in epi
    g = torch.Generator(device=_dev()).manual_seed(Cin * 7 + Cout)
    dw0 = torch.randn(shape, generator=g, device=_dev())
    db0 = torch.randn(Cout, generator=g, device=_dev())
    refs = {}

    def reference(rounded):
        if rounded not in refs:
            refs[rounded] = [torch.nn.grad.conv2d_weight(_nchw(x if rounded else xo.double()), shape,
                                                         _nchw(d if rounded else do.double()), 1, 1)
                             for x, d, xo, do in zip(ops_x, ops_dy, xs, dys)]
        return refs[rounded]
    scale = {}

    def launch(mode):
        if not scale:       # a start of the order of the result
            scale['dw'] = float(sum(reference(True)).std())
            scale['db'] = float(sum(d.double().sum(dim=(0, 1, 2)) for d in dys).pow(2).mean().sqrt())
        dw_start = dw0 * scale['dw']
        db_start = db0 * scale['db']
        dwb, dw = _guarded(Cout * Cin * 9, torch.float32, float('nan'))
        dw.copy_(dw_start.flatten())
        dw = dw.view(shape)
        dbb = db = None
        if dbias:
            dbb, db = _guarded(Cout, torch.float32, float('nan'))
            db.copy_(db_start)
        with _mode(ops, mode):
            if planes:
                ops.wgrad_planes_multi(wd, [dict(x=xp[i], dy=dyp[i], B=B, H=h, W=w) for i, (h, w) in enumerate(levels)],
                                       dw, Cin, Cout, 3)
            else:
                lv = [dict(x_ptr=xs[i].data_ptr(), x_bs=h * w * Cin, dy_ptr=slv[i][0], dy_bs=slv[i][1], B=B, H=h, W=w)
                      for i, (h, w) in enumerate(levels)]
                ops.conv_wgrad_multi(src, lv, dw, db, Cin, Cout, 3, tc=True)
        torch.cuda.synchronize()
        out = dict(dw=dw.double() - dw_start.double(), buffers=[(dwb, Cout * Cin * 9)], bits=[_i32(dw)])
        if dbias:
            out['db'] = db.double() - db_start.double()
            out['buffers'].append((dbb, Cout))
        return out
    s.update(xs=xs, dys=dys, launch=launch, reference=reference,
             dbias_ref=sum(d.double().sum(dim=(0, 1, 2)) for d in dys) if dbias else None)
    return s


# ------------------------------------------------------------------------------------------------
# launches, recorded in a process of their own
# ------------------------------------------------------------------------------------------------

KERNELS = ('conv_planes_kernel', 'conv_tc_kernel', 'wgrad_tc2_multi_kernel', 'wgrad_tc_kernel', 'colsum_kernel')


def _expected_launches(case, sms):
    """[(kernel name, grid or None)] of one case from the mirrors"""
    call, kind, Cin, Cout, B, hw, act, epi = case[1]
    if call == 'planes':
        p = _planes_plan(B, hw, Cin, Cout, sms)
        return [(p['kernel'], p['grid'])]
    if call == 'conv':
        p = _conv_plan(list(hw), B, Cin, Cout)
        return [('conv_tc_kernel<%d,%d,1>(' % (p['BN'], p['stages']), p['grid'])]
    return [(n_, grid) for n_, grid, _ in _wgrad_route(B, hw, Cin, Cout, sms) if n_ != 'colsum_kernel' or 'dbias' in epi]


def _record_launches(out_dir):
    """run every case once in bf16 mode under torch.profiler; write {case id: [(kernel name, grid)]} to
    out_dir/launches.json"""
    from models import _ops as ops
    ops.PRECISION = 'bf16'
    out_dir = pathlib.Path(out_dir)
    rec = {}
    for case in CASES:
        s = _setup(ops, case)
        trace = _launches(lambda: s['launch']('bf16'), out_dir, '_kernel')
        rec[_case_id(case)] = [t for t in trace if any(k + '<' in t[0] or k + '(' in t[0] for k in KERNELS)]
        del s
        torch.cuda.empty_cache()
    with open(out_dir / 'launches.json', 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def launches(tmp_path_factory):
    """the kernel names and grids of every case, recorded by _record_launches in a fresh interpreter (as
    tests/test_gather_path_parity.py's launches fixture)"""
    out = tmp_path_factory.mktemp('single_pass_launches')
    here = os.path.dirname(os.path.abspath(__file__))
    path = [here, os.path.join(REPO, 'oracle'), os.path.join(REPO, 'efficientdet.pytorch_b200'), REPO]
    code = 'import sys; sys.path[:0] = %r; import test_single_pass_parity as T; T._record_launches(%r)' % (path, str(out))
    subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], check=True, cwd=REPO,
                   timeout=1200)
    with open(out / 'launches.json') as f:
        return {k: [(name, tuple(grid)) for name, grid in v] for k, v in json.load(f).items()}


@pytest.fixture()
def ops():
    from models import _ops
    old = _ops.PRECISION
    _ops.PRECISION = 'bf16'
    yield _ops
    _ops.PRECISION = old


def _cat(ts):
    return torch.cat([t.flatten() for t in ts])


def _guards(out, what):
    for buf, n in out['buffers']:
        _check_written(buf, n, what)
    for buf, n, _ in out.get('y_mask', []):
        assert (buf[n:] == 0x5a5a5a5a).all(), ('%s: ReLU bits written past the end' % what)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_single_pass_call(ops, case, launches):
    """one recorded call at its real B, levels and channels: launches, the exact-operand fp64 reference with its
    controls, and the bf16 vs bf16x3 differential check on bf16-exact operands"""
    call, kind, Cin, Cout, B, hw, act, epi = case[1]
    what = '%s %s %s %d->%d B=%d %s %s' % (case[0], call, kind, Cin, Cout, B, act, '+'.join(epi))
    sms = _sms()
    got_l = launches[_case_id(case)]
    want_l = _expected_launches(case, sms)
    print('%s\n  launches %s' % (what, got_l))
    assert len(got_l) == len(want_l) and all(n_ in g_[0] and (grid is None or grid == g_[1])
                                             for (n_, grid), g_ in zip(want_l, got_l)), (got_l, want_l)
    torch.set_num_threads(min(16, os.cpu_count() or 1))

    s = _setup(ops, case)
    one = s['launch']('bf16')
    _guards(one, what)
    three = s['launch']('bf16x3')
    if call == 'wgrad':
        want = s['reference'](True)
        total = sum(want)
        _check_dw(one['dw'], total, what)
        if s['dbias_ref'] is not None:
            e = _rel(one['db'], s['dbias_ref'])
            ctrl_db = _rel(one['db'], s['dbias_ref'] - s['dys'][-1].double().sum(dim=(0, 1, 2)))
            print('  dbias rel err %.2e (bound %.0e), without the last level %.2e' % (e, TOL_SUM, ctrl_db))
            assert e < TOL_SUM and ctrl_db > TOL_SUM, (e, ctrl_db)
        # controls: bf16x3 against the rounded reference, bf16 against the unrounded one, dw without the first 64
        # chunks (4 096 pixels) of P3
        x3 = _rel(three['dw'], total)
        single = _rel(one['dw'], sum(s['reference'](False)))
        (h, w), = s['levels'][:1]
        npx = 64 * WG_MAX_CHUNKS_PER_SPLIT
        d_first = torch.zeros(1, h * w, Cout, device=_dev(), dtype=torch.float64)
        d0 = rn(s['dys'][0][:1]).double().reshape(1, h * w, Cout)
        d_first[:, :npx] = d0[:, :npx]
        first = torch.nn.grad.conv2d_weight(_nchw(rn(s['xs'][0][:1]).double()), (Cout, Cin, 3, 3),
                                            _nchw(d_first.view(1, h, w, Cout)), 1, 1)
        miss = max(_block_errs(one['dw'], total - first))
        print('  controls: bf16x3 vs rounded %.2e, single pass vs unrounded %.2e, without the first 64 chunks of P3 '
              'worst block %.2e' % (x3, single, miss))
        assert x3 > TOL_TC and single > SINGLE_PASS_MIN and miss > TOL_LOCAL, (x3, single, miss)
    else:
        want = s['reference'](True)
        _check(one['levels'], want, what)
        if 'colsum' in one:
            ref_cs = sum(t.sum(dim=(0, 1, 2)) for t in want)
            e = _rel(one['colsum'], ref_cs)
            ctrl_cs = _rel(one['colsum'], ref_cs - want[-1].sum(dim=(0, 1, 2)))
            print('  column sums rel err %.2e (bound %.0e), without the smallest level %.2e' % (e, TOL_SUM, ctrl_cs))
            assert e < TOL_SUM and ctrl_cs > TOL_SUM, (e, ctrl_cs)
        if 'y_mask' in one:
            for (_, _, m), t in zip(one['y_mask'], one['levels']):
                assert torch.equal(m, _mask_words(t, Cout)), 'ReLU bits disagree with the stored output'
        # controls; against the convolution alone where a residual would dilute them
        res = s['res'] or [0] * len(want)
        lin = [t - (r.double() if torch.is_tensor(r) else 0) for t, r in zip(want, res)]
        x3 = _rel(_cat([t - (r.double() if torch.is_tensor(r) else 0) for t, r in zip(three['levels'], res)]), _cat(lin))
        plain = s['reference'](False)
        single = _rel(_cat([t - (r.double() if torch.is_tensor(r) else 0) for t, r in zip(one['levels'], res)]),
                      _cat([t - (r.double() if torch.is_tensor(r) else 0) for t, r in zip(plain, res)]))
        miss = max(_rel(g_, w_) for g_, w_ in zip(one['levels'], want[:-1] + [torch.zeros_like(want[-1])]))
        print('  controls: bf16x3 vs rounded %.2e, single pass vs unrounded %.2e, without the smallest level %.2e'
              % (x3, single, miss))
        assert x3 > TOL_TC and single > SINGLE_PASS_MIN and miss > TOL_LOCAL, (x3, single, miss)
    del one, three, s
    torch.cuda.empty_cache()

    # differential check on bf16-exact operands
    s = _setup(ops, case, exact=True)
    one = s['launch']('bf16')
    a = s['launch']('bf16x3')
    b = s['launch']('bf16x3') if call == 'wgrad' or 'colsum' in epi else None    # the atomics-order floor
    _guards(one, what)
    if call == 'wgrad':
        det = all(grid is None or grid[2] == 1 for _, grid in want_l if grid is not None)
        if det:
            assert all(torch.equal(u, v) for u, v in zip(one['bits'], a['bits'])), 'bf16 and bf16x3 dw differ'
            print('  differential: dw bit-identical (every launch in one split)')
        else:
            floor = _rel(a['dw'], b['dw'])
            d = _rel(one['dw'], a['dw'])
            print('  differential: dw bf16 vs bf16x3 %.2e, bf16x3 vs bf16x3 %.2e (bound %.2e)'
                  % (d, floor, max(2 * floor, DIFF_FLOOR)))
            assert d <= max(2 * floor, DIFF_FLOOR), (d, floor)
        if 'db' in one:
            floor, d = _rel(a['db'], b['db']), _rel(one['db'], a['db'])
            print('  differential: dbias %.2e, bf16x3 vs bf16x3 %.2e' % (d, floor))
            assert d <= max(2 * floor, DIFF_FLOOR), (d, floor)
    else:
        same = all(torch.equal(u, v) for u, v in zip(one['bits'], a['bits']))
        assert same, 'bf16 and bf16x3 outputs differ on bf16-exact operands'
        msg = '  differential: outputs%s bit-identical' % (' and ReLU bits' if 'y_mask' in one else '')
        if 'colsum' in one:
            floor, d = _rel(a['colsum'], b['colsum']), _rel(one['colsum'], a['colsum'])
            msg += '; column sums %.2e, bf16x3 vs bf16x3 %.2e' % (d, floor)
            assert d <= max(2 * floor, DIFF_FLOOR), (d, floor)
        print(msg)
