"""Kernel-level fp64 parity of the MBConv backbone at the D1-D3 and D5-D7 input sizes.

  pw_gemm_kernel       the expand conv's data gradient from an fp32 operand (expand_dgrad_fp32), with and without the
                       skip block's residual, and the expand forward with three images in one m-tile (pw_gemm.cu)
  pw_wgrad_kernel      the expand conv's weight gradient with dy in fp32, and the NB = 2 instances of the other modes
  dw_fwd_fused_kernel, dw_bwd_fused_kernel   a last 16-channel group with idle lanes (C % 16 != 0, dw_fused.cu)
  stem_fwd_px_kernel, bnact_bwd_kernel, stem_wgrad_kernel   the stem at native sizes (stem.cu)
  MBConvFn             forward and backward composed on the fp32 data-gradient route
  the SE gate and spatial_reduce_act at the pyramids' shapes

MBConvFn.backward hands the depthwise input gradient to the expand conv as bf16 hi/lo planes when its map has a TMA
pixel box (ops.planes_ok: W <= 64 or W % 64 == 0, and a box of a multiple of 16 pixels); otherwise
dw_bwd_fused_kernel writes it in fp32 and pw_wgrad_kernel and pw_gemm_kernel read it in fp32.  bench.CONFIGS (d0, d4,
d7) has a pixel box on every backbone map, so the second route never runs there.  At the reference's input sizes it
carries most expand blocks (the same at every B = 1..8):

  model  input  backbone  expand blocks on the fp32 route  of them skip blocks (residual = dy)
  D1      640     B1           20 of 21                         15
  D2      768     B2            4 of 21                          3
  D3      896     B3           23 of 24                         18
  D5     1280     B5           30 of 36                         26
  D6     1408     B6           41 of 42                         36
  D7     1536     B6            8 of 42                          7

A depthwise CTA owns 16 channels (kCVc = 4 float4 vectors); when C % 16 != 0 the last group has idle lanes.  That
happens only in stage-1 blocks without BN0 on the largest maps: C 40 and 24 at 448x448 (B3), 24 at 640x640 (B5), 56 at
704x704 and 768x768 (B6), up to 8 tiles per CTA.  The stem's weight gradient strides one CTA over up to 70 row
segments (D7, B = 8).  This file

  * walks every MBConv block of D1-D3 and D5-D7 at B = 1..8, forward and backward, with the launcher mirrors of
    tests/test_pointwise_se_parity.py (_pwg_plan) and tests/test_benchmark_plans.py (_pw_plan, _dw_plan, _stem_plan),
    checks the table above against the library, and checks that the cases below reach every pw_gemm plan class, every
    pw_wgrad (mode, NB) pair, every partial-group depthwise class and the stem's longest segment ranges that the
    existing cases do not reach, and that removing any case loses one (test_cases_reach_pyramid_plans);
  * records every launch once under torch.profiler in a fresh interpreter (the launches fixture) and compares kernel
    name, grid and (pw_gemm) dynamic shared memory with the mirrors;
  * holds each call, into NaN-filled outputs with a guard after every output buffer, to float64 on the device.

Bounds (norm-relative error ||got - want|| / ||want||), as the sibling files:
  TOL_TC    = 3e-5  a whole bf16x3 output
  TOL_ROW   = 1e-4  each image and each 64-column block of a pw_gemm output, each row of a pointwise weight gradient
  TOL_DW    = 5e-5  the fp32 depthwise kernels: whole tensors, each image's SE mean, each tap of dW, the BN affines
  TOL_EXACT = 5e-6  fp32 element-wise outputs of the stem and of bnact_bwd, the SE gate
  TOL_SUM   = 2e-5  sums over many atomic blocks (stem weight gradient and BN affines, spatial_reduce_act)
  TOL_MB_FWD = 1e-4, TOL_MB_GRAD = 2e-4  the composed block
Negative controls, each of which must exceed the bound it guards: the last 64-column block without its last k-block
(per block), hi*hi bf16 products only (whole), the output without the residual (whole); the weight gradient without
the pixels one CTA accumulates (whole and per row); one image's SE mean without one forward tile (per image); dW
without the output gradient of one backward tile (per tap); the stem's dW without the last row segment (TOL_SUM); the
composed block's input gradient against a reference with a bf16-rounded expand weight, and without the skip path's dy
(TOL_MB_GRAD); the SE gate's and spatial_reduce_act's controls of tests/test_pointwise_se_parity.py.

Measured on an H100 80GB HBM3 at 700 W (worst case of each test):
  pw_gemm_kernel, fp32 route and expand forward   whole tensor 3.7e-6 .. 6.5e-6, worst image 6.6e-6, worst 64-column
                                                  block 6.6e-6 (1920 -> 320 at 5x5, KB 30, three images per tile)
  pw_wgrad_kernel, plain 144 -> 864 at 96x96, B 4 1.46e-5 whole, 1.72e-5 worst row (4 096 pixels per CTA); planes
                                                  and project at NB 2 4.5e-6 whole, 7.4e-6 worst row
  depthwise, C 24, 40, 56                         z1 5.8e-8, dx 1.1e-7, SE mean 2.9e-7 (per image), dW 1.05e-6 (per
                                                  tap), BN affines 6.7e-7; the last partial group alone no worse:
                                                  dx 1.1e-7, mean 4.2e-7, dW 6.7e-7, affines 6.9e-7
  stem at 896 (C0 40, B 8) and 1536 (C0 56, B 8)  z, y, dz 1.34e-7; dW 7.8e-7, dgamma, dbeta 4.6e-7 (70 segments per
                                                  CTA)
  MBConvFn on the fp32 route                      output 6.2e-6, input gradient 7.9e-6, parameter gradients 9.4e-6
  SE gate, every new (B, C, S)                    9.2e-7
  spatial_reduce_act                              4.4e-7 per image
The weakest controls: hi*hi only 2.3e-3, the last k-block missing from one column block 1.5e-1, the residual missing
6.5e-1, the weight gradient without one CTA's pixels 3.5e-1, one image's mean without a forward tile 5.2e-4 (10x
TOL_DW), dW without a backward tile 1.8e-2, the stem's dW without its last segment 2.8e-3, the composed block with a
bf16 expand weight 1.4e-3, the SE gate's 4.6e-1, spatial_reduce_act without one row block 1.1e-1.  No kernel needed a
change."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O
from test_benchmark_plans import BN_EPS, SMS, TOL_DW, TOL_EXACT, TOL_ROW, TOL_SUM, TOL_TC, _dw_out, _dw_plan, \
    _dw_reference, _pw_plan, _stem_out, _stem_plan
from test_benchmark_plans import PW_CASES as BENCH_WGRAD_CASES, STEM_CASES as BENCH_STEM_CASES
from test_planes_path_parity import _box
from test_planes_path_parity import ops  # noqa: F401  (the bf16x3 fixture)
from test_pointwise_se_parity import PW_CASES as BENCH_PW_CASES, TOL_MB_FWD, TOL_MB_GRAD, _case_call, _plan_of, \
    _pw_class, _pw_errs, _pwg_plan, _rel, _row_grid, _se_shapes, _sra_cases, _sra_setup, _trace
# the SE gate and spatial_reduce_act checks, called at the pyramids' shapes (underscored: not collected here again)
from test_pointwise_se_parity import test_se_gate as _se_gate_check, test_spatial_reduce_act as _sra_check

GUARD = 4096                    # elements after every output buffer, NaN (stored outputs) or 0 (accumulated ones)
# (detector, input size) of the reference's configs whose backbones take the fp32 route (utils/config_eff.py)
PYRAMIDS = {'d1_640': ('efficientdet-d1', 640), 'd2_768': ('efficientdet-d2', 768), 'd3_896': ('efficientdet-d3', 896),
            'd5_1280': ('efficientdet-d5', 1280), 'd6_1408': ('efficientdet-d6', 1408),
            'd7_1536': ('efficientdet-d7', 1536)}
FP32_ROUTE = {'d1_640': (20, 21, 15), 'd2_768': (4, 21, 3), 'd3_896': (23, 24, 18), 'd5_1280': (30, 36, 26),
              'd6_1408': (41, 42, 36), 'd7_1536': (8, 42, 7)}
BATCHES = range(1, 9)


def _dev():
    return torch.device('cuda:0')


# ------------------------------------------------------------------------------------------------
# the walk
# ------------------------------------------------------------------------------------------------

def _walk(geo, B):
    """every call of one training step of the backbone of `geo` at batch B: pw_gemm calls (block, route, shape
    (B, H, W, Cin, Cout), skip), pw_wgrad calls (block, mode, shape), depthwise launches (block, dir, k, s, BN0, C, H, W),
    the stem (C0, size), SE gates (B, C, S) and spatial_reduce_act calls (B, HW, C)"""
    net, size = PYRAMIDS[geo]
    cfg = O.make_config(net)
    H, W = _stem_out(size, size)
    out = dict(pw=[], wgrad=[], dw=[], se=[], sra=[], stem=(cfg['stem'], size))
    for i, blk in enumerate(cfg['blocks']):
        mid = blk['cin'] * blk['e']
        expand = blk['e'] != 1
        Ho, Wo = _dw_out(blk['k'], blk['s'], H, W)
        planes = expand and mid % 8 == 0 and _box(B, H, W) is not None      # MBConvFn.backward: ops.planes_ok
        if expand:
            out['pw'].append(dict(block=i, route='expand_fwd', shape=(B, H, W, blk['cin'], mid), skip=False))
            out['wgrad'].append(dict(block=i, mode='planes' if planes else 'plain', shape=(B, H, W, blk['cin'], mid)))
        out['pw'].append(dict(block=i, route='project_fwd', shape=(B, Ho, Wo, mid, blk['cout']), skip=blk['skip']))
        out['pw'].append(dict(block=i, route='project_dgrad', shape=(B, Ho, Wo, blk['cout'], mid), skip=False))
        out['wgrad'].append(dict(block=i, mode='project', shape=(B, Ho, Wo, mid, blk['cout'])))
        if expand:
            out['pw'].append(dict(block=i, route='expand_dgrad_planes' if planes else 'expand_dgrad_fp32',
                                  shape=(B, H, W, mid, blk['cin']), skip=blk['skip']))
        for d in ('fwd', 'bwd'):
            out['dw'].append(dict(block=i, dir=d, k=blk['k'], s=blk['s'], pre=expand, C=mid, H=H, W=W))
        out['se'].append((B, mid, blk['sq']))
        out['sra'].append((B, Ho * Wo, mid))
        H, W = Ho, Wo
    return out


def _pw_key(route, plan, skip):
    """a pw_gemm plan class; on the fp32 data-gradient route with or without the residual"""
    return _pw_class(route, plan), (skip if route == 'expand_dgrad_fp32' else None)


def _find(geo, block, B, kind, **match):
    calls = [c for c in _walk(geo, B)[kind] if c['block'] == block and all(c[k] == v for k, v in match.items())]
    assert len(calls) == 1, (geo, block, B, kind, match, calls)
    return calls[0]


# ------------------------------------------------------------------------------------------------
# the GPU cases
# ------------------------------------------------------------------------------------------------

# pw_gemm: (pyramid, block, route, B), each at the walk's own shape; per plan class of the fp32 route a skip block
# (residual = dy) and a block without skip, each at the smallest B and map that reach it
PW_CASES = [
    ('d1_640', 3, 'expand_dgrad_fp32', 1), ('d1_640', 8, 'expand_dgrad_fp32', 1),     # 144->24 160^2, 240->40 80^2
    ('d2_768', 6, 'expand_dgrad_fp32', 1), ('d2_768', 8, 'expand_dgrad_fp32', 1),     # 288->48 96^2, streamed weights
    ('d1_640', 9, 'expand_dgrad_fp32', 1), ('d1_640', 21, 'expand_dgrad_fp32', 1),    # NB 2: 480->80 40^2, 1152->192
    ('d1_640', 22, 'expand_dgrad_fp32', 2), ('d1_640', 21, 'expand_dgrad_fp32', 2),   # ... two images per m-tile
    ('d1_640', 22, 'expand_dgrad_fp32', 3), ('d1_640', 21, 'expand_dgrad_fp32', 6),   # ... three or more
    ('d1_640', 22, 'expand_fwd', 3),                                                  # 320->1920 5^2, NB 2, three
]
# pw_wgrad: (pyramid, block, mode, B).  The longest plain K range (4 096 pixels per CTA at NB 2) and the smallest
# layers of the NB = 2 instances of planes and project, which tests/test_benchmark_plans.py's cases do not reach
WGRAD_CASES = [('d7_1536', 23, 'plain', 4), ('d2_768', 17, 'planes', 1), ('d1_640', 21, 'project', 1)]
# depthwise with a partial last channel group: (pyramid, block, B).  C 24 and C 56 at the smallest B with 8 tiles per
# CTA (the cap), C 40 at the smallest B with a partial last group of several tiles
DW_CASES = [('d3_896', 0, 4), ('d5_1280', 1, 7), ('d6_1408', 0, 3)]
# stem: (pyramid, B).  TPG 9 (C0 40) and TPG 14 (C0 56) at the walk's most segments per CTA
STEM_CASES = [('d3_896', 8), ('d7_1536', 8)]
# the composed block: (pyramid, block, B, drop-connect): a skip block and a block without skip, both without a box
MB_CASES = [('d1_640', 4, 2, True), ('d1_640', 5, 1, False)]


def _walk_all():
    return {(geo, B): _walk(geo, B) for geo in PYRAMIDS for B in BATCHES}


def _pw_call(case):
    geo, block, route, B = case
    return _find(geo, block, B, 'pw', route=route)


def _wgrad_call(case):
    geo, block, mode, B = case
    return _find(geo, block, B, 'wgrad', mode=mode)


def _dw_case(case):
    """(k, s, BN0, C, H, W, B) of a depthwise case"""
    geo, block, B = case
    c = _find(geo, block, B, 'dw', dir='fwd')
    return c['k'], c['s'], c['pre'], c['C'], c['H'], c['W'], B


def _stem_case(case):
    geo, B = case
    C0, size = _walk(geo, B)['stem']
    return C0, size, size, B


def _se_cases(walks):
    """{(C, S): [B]} of the walk's SE gates not among tests/test_pointwise_se_parity.py's shapes"""
    old = set(_se_shapes())
    out = {}
    for w in walks.values():
        for B, C, S in w['se']:
            if (B, C, S) not in old:
                out.setdefault((C, S), set()).add(B)
    return {k: sorted(v) for k, v in sorted(out.items())}


def _sra_pyramid_cases(walks):
    """the walk's spatial_reduce_act with the most rows per block, and with the most channel chunks at the smallest map"""
    calls = sorted({t for w in walks.values() for t in w['sra']})
    rows = max(calls, key=lambda t: _row_grid(t[1], t[2] // 4, t[0], SMS)[1])
    chunks = max(calls, key=lambda t: (_row_grid(t[1], t[2] // 4, t[0], SMS)[0][1], -t[0] * t[1]))
    return [rows, chunks]


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_fp32_route_table():
    """the table of the docstring from the walk, and ops.planes_ok's pixel box from the library
    (effdet_wgrad_tc_geometry_ok) against the mirror _box on every backbone map at B = 1..8"""
    import __graft_entry__ as entry
    entry.build()
    from models import _native as N
    lib = N.load()
    for geo in PYRAMIDS:
        for B in BATCHES:
            w = _walk(geo, B)
            ex = [c for c in w['pw'] if c['route'].startswith('expand_dgrad')]
            fp = [c for c in ex if c['route'] == 'expand_dgrad_fp32']
            assert (len(fp), len(ex), sum(c['skip'] for c in fp)) == FP32_ROUTE[geo], (geo, B)
            maps = {c['shape'][1:3] for c in w['pw']}
            for h, ww in maps:
                assert bool(lib.effdet_wgrad_tc_geometry_ok(B, h, ww)) == (_box(B, h, ww) is not None), (geo, B, h, ww)


def test_mirrors():
    """the launchers' arithmetic on the figures that motivated the cases (132 SMs)"""
    p = _pwg_plan(*_pw_call(('d1_640', 22, 'expand_fwd', 3))['shape'], False, SMS)
    assert (p['NB'], p['bres'], p['images'], p['KB'], p['ntn']) == (2, False, 3, 5, 15)
    p = _pwg_plan(*_pw_call(('d1_640', 9, 'expand_dgrad_fp32', 1))['shape'], False, SMS)
    assert (p['NB'], p['KB'], p['ntn'], p['bres']) == (2, 8, 1, False)
    w = _wgrad_call(WGRAD_CASES[0])
    assert w['shape'] == (4, 96, 96, 144, 864)
    assert _pw_plan(*w['shape'], SMS)['pixels'] == 4096 and _pw_plan(*w['shape'], SMS)['NB'] == 2
    assert [_dw_case(c)[3] for c in DW_CASES] == [40, 24, 56]
    p = _dw_plan('fwd', 3, 1, 56, 704, 704, 3)
    assert (p['ntiles'], p['tpc'], p['grid']) == (1936, 8, (4, 242, 3))
    assert _stem_plan(8, 1536, 1536, 56, SMS)['segs_per_cta'] == 70
    assert _stem_plan(8, 896, 896, 40, SMS)['tpg'] == 9
    for geo, block, B, drop in MB_CASES:
        c = _find(geo, block, B, 'pw', route='expand_dgrad_fp32')
        assert c['skip'] == drop and _box(*c['shape'][:3]) is None


def _missing(pw_cases, wgrad_cases, dw_cases, stem_cases, walks):
    """what the walk reaches that neither these cases nor the existing files' cases reach"""
    miss = []
    # pw_gemm plan classes
    bench = {_pw_key(c[2], _plan_of(_case_call(c)), False) for c in BENCH_PW_CASES}
    want = set()
    for w in walks.values():
        for c in w['pw']:
            want.add(_pw_key(c['route'], _pwg_plan(*c['shape'], c['route'] == 'expand_dgrad_planes', SMS), c['skip']))
    got = bench.copy()
    for case in pw_cases:
        c = _pw_call(case)
        got.add(_pw_key(c['route'], _pwg_plan(*c['shape'], False, SMS), c['skip']))
    miss += [('pw_gemm', k) for k in sorted(want - got, key=str)]
    # pw_wgrad (mode, NB) pairs and the longest plain pixel range per CTA
    walk_wg = [(c['mode'], _pw_plan(*c['shape'], SMS)) for w in walks.values() for c in w['wgrad']]
    case_wg = [(c[5], _pw_plan(*c[:5], SMS)) for c in BENCH_WGRAD_CASES.values()]
    case_wg += [(m, _pw_plan(*_wgrad_call(case)['shape'], SMS)) for case in wgrad_cases for m in [case[2]]]
    miss += [('pw_wgrad', k) for k in sorted({(m, p['NB']) for m, p in walk_wg} - {(m, p['NB']) for m, p in case_wg})]
    longest = max(p['pixels'] for m, p in walk_wg if m == 'plain')
    mine = [_pw_plan(*_wgrad_call(c)['shape'], SMS) for c in wgrad_cases if c[2] == 'plain']
    if max((p['pixels'] for p in mine), default=0) < longest:
        miss.append(('pw_wgrad plain pixels per CTA', longest))
    # depthwise with C % 16 != 0: every (direction, k, s, BN0, SMALL) class and channel count, the most tiles per CTA,
    # a partial last tile group of several tiles
    walk_dw, case_dw = [], []
    for (geo, B), w in walks.items():
        for c in w['dw']:
            if c['C'] % 16:
                walk_dw.append((c['dir'], c['k'], c['s'], c['pre'], c['C'],
                                _dw_plan(c['dir'], c['k'], c['s'], c['C'], c['H'], c['W'], B)))
    for case in dw_cases:
        k, s, pre, C, H, W, B = _dw_case(case)
        for d in ('fwd', 'bwd'):
            case_dw.append((d, k, s, pre, C, _dw_plan(d, k, s, C, H, W, B)))

    def dw_feats(launches):
        f = {('class', d, k, s, pre, p['small']) for d, k, s, pre, C, p in launches}
        f |= {('C', C) for *_, C, p in launches}
        f |= {('tiles per CTA', max(p['tpc'] for *_, p in launches))}
        f |= {('partial group of several tiles',) for *_, p in launches if p['partial'] and p['tpc'] > 1}
        return f
    miss += [('dw', k) for k in sorted(dw_feats(walk_dw) - dw_feats(case_dw), key=str)]
    # stem: the most segments per CTA of each TPG instantiation
    walk_st, case_st = {}, {}
    for (geo, B), w in walks.items():
        C0, size = w['stem']
        p = _stem_plan(B, size, size, C0, SMS)
        walk_st[p['tpg']] = max(walk_st.get(p['tpg'], 0), p['segs_per_cta'])
    for C0, H, W, B in list(BENCH_STEM_CASES.values()) + [_stem_case(c) for c in stem_cases]:
        p = _stem_plan(B, H, W, C0, SMS)
        case_st[p['tpg']] = max(case_st.get(p['tpg'], 0), p['segs_per_cta'])
    miss += [('stem', t, n) for t, n in sorted(walk_st.items()) if case_st.get(t, 0) < n]
    return miss


def test_cases_reach_pyramid_plans():
    """the cases reach every plan class of the walk that the existing cases do not, and each case is needed: without
    it something is lost; every composed case takes the fp32 route, and the SE and spatial_reduce_act cases are new"""
    walks = _walk_all()
    lists = [PW_CASES, WGRAD_CASES, DW_CASES, STEM_CASES]
    assert _missing(*lists, walks) == []
    for j, lst in enumerate(lists):
        for i in range(len(lst)):
            fewer = list(lists)
            fewer[j] = lst[:i] + lst[i + 1:]
            assert _missing(*fewer, walks), ('not needed', lst[i])
    # the plan classes new to pw_gemm here: five on the fp32 route, and the expand forward with NB 2 and three images
    # in one m-tile
    bench = {_pw_class(c[2], _plan_of(_case_call(c))) for c in BENCH_PW_CASES}
    new = {_pw_class(c[2], _pwg_plan(*_pw_call(c)['shape'], False, SMS)) for c in PW_CASES} - bench
    assert sorted(r for r, *_ in new) == ['expand_dgrad_fp32'] * 5 + ['expand_fwd'], new
    # the longest plain range is the cap, and no walk layer exceeds it
    assert max(_pw_plan(*c['shape'], SMS)['pixels'] for w in walks.values() for c in w['wgrad']) == 4096
    # composed cases on the fp32 route, one with skip and drop-connect, one without skip
    assert {drop for *_, drop in MB_CASES} == {True, False}
    se = _se_cases(walks)
    assert se and not set(_se_shapes()) & {(B, C, S) for (C, S), bs in se.items() for B in bs}
    sra = _sra_pyramid_cases(walks)
    assert not set(sra) & set(_sra_cases()), sra
    assert sra == [(8, 589824, 32), (1, 121, 3456)], sra


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _sms():
    return torch.cuda.get_device_properties(_dev()).multi_processor_count


def _gen(seed):
    return torch.Generator(device=_dev()).manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device=_dev())


def _rand(g, *shape):
    return torch.rand(*shape, generator=g, device=_dev())


def _swish(x):
    return x * torch.sigmoid(x)


class _Out:
    """an output buffer followed by GUARD elements of its fill: NaN for stored outputs (an element left unwritten fails
    its bound), 0 for outputs the kernels accumulate into (any stray atomic changes the guard)"""

    def __init__(self, shape, fill):
        n = 1
        for d in shape:
            n *= d
        self.buf = torch.full((n + GUARD,), fill, device=_dev())
        self.n, self.fill = n, fill
        self.t = self.buf[:n].view(shape)

    def guard_ok(self):
        tail = self.buf[self.n:]
        return bool(torch.isnan(tail).all()) if self.fill != self.fill else bool((tail == self.fill).all())


class _guarded:
    """ops._empty and ops._zeros hand out _Out buffers inside the block (NaN- and zero-filled); .outs lists them"""

    def __init__(self, ops):
        self.ops, self.outs = ops, []

    def __enter__(self):
        self.old = self.ops._empty, self.ops._zeros

        def make(fill):
            def alloc(shape, like):
                o = _Out(tuple(shape), fill)
                self.outs.append(o)
                return o.t
            return alloc
        self.ops._empty, self.ops._zeros = make(float('nan')), make(0.0)
        return self

    def __exit__(self, *exc):
        self.ops._empty, self.ops._zeros = self.old


def _check_guards(outs, what):
    assert outs and all(o.guard_ok() for o in outs), ('%s: written past the end of an output' % what)


# ------------------------------------------------------------------------------------------------
# the calls of the GPU tests, and their launches recorded in a process of their own
# ------------------------------------------------------------------------------------------------

def _pwg_setup(ops, case):
    """inputs and the pw_gemm call of `case` as MBConvFn makes it: launch() -> (y, guarded buffers)"""
    c = _pw_call(case)
    route, (B, H, W, Cin, Cout), skip = c['route'], c['shape'], c['skip']
    g = _gen(31 + PW_CASES.index(case))
    x = _randn(g, B, H, W, Cin)
    if route == 'expand_fwd':
        w = _randn(g, Cout, Cin, 1, 1) * (1.5 / Cin ** 0.5)
        wp, wtc, weight = ops.pack_conv(w)[0], ops.tc_packs(w)[0], w.view(Cout, Cin).double()
    else:
        # the expand weight We [mid, cin]: the data gradient runs mid -> cin on its dgrad pack, the residual is dy
        w = _randn(g, Cin, Cout, 1, 1) * (1.5 / Cin ** 0.5)
        wp, wtc, weight = ops.pack_conv(w)[1], ops.tc_packs(w)[1], w.view(Cin, Cout).t().double()
    assert wtc is not None
    res = _randn(g, B, H, W, Cout) if skip else None

    def launch():
        with _guarded(ops) as gd:
            y = ops.conv2d(x, wp, Cout, 1, residual=res, w_tc=wtc)
        return y, gd.outs
    return dict(call=c, B=B, H=H, W=W, Cin=Cin, Cout=Cout, M=B * H * W, x=x, weight=weight, res=res, launch=launch)


def _wgrad_setup(ops, case):
    """inputs of a pw_wgrad case and launch(dw), which adds dy^T act(x) to dw as MBConvFn.backward calls it"""
    c = _wgrad_call(case)
    mode, (B, H, W, Cin, Cout) = c['mode'], c['shape']
    g = _gen(Cin * 1000 + Cout + B)
    x = _randn(g, B, H, W, Cin)
    dy = _randn(g, B, H, W, Cout)
    sc, sh = _rand(g, Cin) + 0.5, _randn(g, Cin) * 0.3
    gate = _rand(g, B, Cin)
    planes = None
    if mode == 'planes':
        assert ops.planes_ok(B, H, W, Cout)
        hi = dy.to(torch.bfloat16)
        planes = torch.stack([hi, (dy - hi.float()).to(torch.bfloat16)]).contiguous()
    elif mode == 'plain':
        assert not ops.planes_ok(B, H, W, Cout)

    def launch(dw):
        if mode == 'planes':
            ops.conv_wgrad_raw(x, ops.N.f32(x), H * W * Cin, None, H * W * Cout, dw, None, B, H, W, Cin, Cout, 1, tc=True,
                               dy_planes=planes)
        elif mode == 'project':
            ops.conv_wgrad(x, dy, dw, None, 1, a_scale=gate, tc=True, in_scale=sc, in_shift=sh)
        else:
            ops.conv_wgrad(x, dy, dw, None, 1, tc=True)

    def act(b, rows=slice(None)):
        a = x[b].reshape(-1, Cin)[rows].double()
        if mode == 'project':
            a = _swish(a * sc.double() + sh.double()) * gate[b].double()
        return a
    return dict(mode=mode, B=B, H=H, W=W, Cin=Cin, Cout=Cout, g=g, dy=dy, act=act, launch=launch)


def _fold(bn, i):
    rstd = 1.0 / torch.sqrt(bn[i]['v'] + BN_EPS)
    sc = bn[i]['g'] * rstd
    return [t.contiguous() for t in (sc, bn[i]['b'] - bn[i]['m'] * sc, bn[i]['m'], rstd)]


def _dw_setup(case):
    """inputs and guarded outputs of a depthwise case; fwd() and bwd() launch the fused kernels as MBConvFn does"""
    from models import _native as N
    k, s, pre, C, H, W, B = _dw_case(case)
    pt = (k - 1) // 2 if s == 1 else (0 if k == 3 else 1)
    Ho, Wo = _dw_out(k, s, H, W)
    g = _gen(k * 100 + s * 10 + C + H + B)
    x = _randn(g, B, H, W, C)
    wd = _randn(g, C, 1, k, k) / k
    bn = [dict(g=_rand(g, C) + 0.5, b=_randn(g, C) * 0.3, m=_randn(g, C) * 0.3, v=_rand(g, C) + 0.5) for _ in range(2)]
    gate = _rand(g, B, C)
    dq = _randn(g, B, Ho, Wo, C)
    dmean = _randn(g, B, C)
    sc0, sh0, mu0, rs0 = _fold(bn, 0)
    sc1, sh1, mu1, rs1 = _fold(bn, 1)
    wkkc = wd.view(C, k * k).t().contiguous()
    nan = float('nan')
    o = dict(z1=_Out((B, Ho, Wo, C), nan), mean=_Out((B, C), 0.0), dx=_Out((B, H, W, C), nan),
             dw=_Out((C, 1, k, k), 0.0), dgamma1=_Out((C,), 0.0), dbeta1=_Out((C,), 0.0))
    if pre:
        o.update(dgamma0=_Out((C,), 0.0), dbeta0=_Out((C,), 0.0))

    def p(name):
        return N.f32(o[name].t) if name in o else None
    fa = N.DwFwdArgs(N.f32(x), N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(wkkc), N.f32(sc1),
                     N.f32(sh1), p('z1'), p('mean'), B, H, W, C, k, s, pt, pt, Ho, Wo, 1.0 / (Ho * Wo))
    ba = N.DwBwdArgs(N.f32(dq), p('z1'), N.f32(gate), N.f32(dmean), N.f32(sc1), N.f32(sh1), N.f32(mu1), N.f32(rs1),
                     N.f32(x), N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(mu0) if pre else None,
                     N.f32(rs0) if pre else None, N.f32(wkkc), p('dx'), p('dw'), p('dgamma1'), p('dbeta1'), p('dgamma0'),
                     p('dbeta0'), 1.0 / (Ho * Wo), B, H, W, C, k, s, pt, pt, Ho, Wo, None)
    return dict(k=k, s=s, pre=pre, C=C, H=H, W=W, B=B, Ho=Ho, Wo=Wo, x=x, wd=wd, bn=bn, gate=gate, dq=dq, dmean=dmean,
                sc1=sc1, sh1=sh1, out=o, fwd=lambda: N.call('effdet_dwconv_fwd_fused', x, fa),
                bwd=lambda: N.call('effdet_dwconv_bwd_fused', x, ba))


def _stem_setup(case):
    """inputs and guarded outputs of a stem case: fwd() (effdet_stem_fwd), bnact() (effdet_bnact_bwd, SWISH), wgrad()"""
    from models import _native as N
    from test_benchmark_plans import _bn_params
    C0, H, W, B = _stem_case(case)
    Ho, Wo = _stem_out(H, W)
    g = _gen(C0 * 7 + H + W + B)
    x = _randn(g, B, 3, H, W)
    w = _randn(g, C0, 3, 3, 3) * (1.5 / 27 ** 0.5)
    gamma, beta, mu, var, scale, shift, rstd = _bn_params(g, C0)
    dy = _randn(g, B, Ho, Wo, C0)
    nan = float('nan')
    o = dict(z=_Out((B, Ho, Wo, C0), nan), y=_Out((B, Ho, Wo, C0), nan), dz=_Out((B, Ho, Wo, C0), nan),
             dgamma=_Out((C0,), 0.0), dbeta=_Out((C0,), 0.0), dw=_Out((C0, 3, 3, 3), 0.0))
    f = {n: N.f32(v.t) for n, v in o.items()}

    def fwd():
        N.call('effdet_stem_fwd', x, N.f32(x), N.f32(w), N.f32(scale), N.f32(shift), f['z'], f['y'], B, H, W, C0)

    def bnact():                # ops.bnact_bwd's call, into guarded buffers
        from models import _ops as ops
        a = N.BnActBwdArgs(N.f32(dy), f['z'], f['dz'], N.f32(scale), N.f32(shift), N.f32(mu), N.f32(rstd), f['dgamma'],
                           f['dbeta'], None, None, None, 1.0 / (Ho * Wo), B, Ho * Wo, C0, ops.ACT_SWISH)
        N.call('effdet_bnact_bwd', x, a)

    def wgrad():
        N.call('effdet_stem_wgrad', x, N.f32(x), f['dz'], f['dw'], B, H, W, C0)
    return dict(C0=C0, H=H, W=W, B=B, Ho=Ho, Wo=Wo, x=x, w=w, gamma=gamma, beta=beta, mu=mu, var=var, dy=dy, out=o,
                fwd=fwd, bnact=bnact, wgrad=wgrad)


def _record_launches(out_dir):
    """run every call of the GPU tests once under torch.profiler; write {case: [(name, grid, shared memory)]} to
    out_dir/launches.json"""
    from models import _ops as ops
    ops.PRECISION = 'bf16x3'
    rec = {}
    for B, HW, C in _sra_pyramid_cases(_walk_all()):
        s = _sra_setup(B, HW, C)
        rec['sra %d %d %d' % (B, HW, C)] = _trace(s['launch'], out_dir, 'spatial_reduce_kernel')
        del s
    for case in PW_CASES:
        s = _pwg_setup(ops, case)
        rec[str(case)] = _trace(s['launch'], out_dir, 'pw_gemm_kernel')
    for case in WGRAD_CASES:
        s = _wgrad_setup(ops, case)
        dw = torch.zeros(s['Cout'], s['Cin'], 1, 1, device=_dev())
        rec[str(case)] = _trace(lambda: s['launch'](dw), out_dir, 'pw_wgrad_kernel')
    for case in DW_CASES:
        s = _dw_setup(case)
        rec[str(case) + ' fwd'] = _trace(s['fwd'], out_dir, 'dw_fwd_fused_kernel')
        rec[str(case) + ' bwd'] = _trace(s['bwd'], out_dir, 'dw_bwd_fused_kernel')
        del s
    for case in STEM_CASES:
        s = _stem_setup(case)
        s['fwd']()
        s['bnact']()
        rec[str(case)] = _trace(s['wgrad'], out_dir, 'stem_wgrad_kernel')
        del s
    with open(os.path.join(str(out_dir), 'launches.json'), 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def launches(tmp_path_factory):
    """the kernel names, grids and shared memory of every call below, recorded by _record_launches in a fresh
    interpreter: a CUDA activity trace in a long test process can miss this library's kernels"""
    out = tmp_path_factory.mktemp('backbone_pyramid_launches')
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    path = [here, os.path.join(repo, 'oracle'), os.path.join(repo, 'efficientdet.pytorch_b200'), repo]
    code = 'import sys; sys.path[:0] = %r; import test_backbone_pyramid_parity as T; T._record_launches(%r)' % (
        path, str(out))
    subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], check=True, cwd=repo,
                   timeout=1200)
    with open(out / 'launches.json') as f:
        return {k: [(n, tuple(grid), smem) for n, grid, smem in v] for k, v in json.load(f).items()}


def _check_launch(ln, name, grid, what, smem=None):
    print('  %s launch: %s' % (what, ln))
    assert len(ln) == 1 and name in ln[0][0] and ln[0][1] == grid, (what, ln, name, grid)
    assert smem is None or ln[0][2] == smem, (what, ln, smem)


# ------------------------------------------------------------------------------------------------
# 1. pw_gemm_kernel on the expand conv's fp32 data-gradient route
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', PW_CASES, ids=['%s-%d-%s-B%d' % c for c in PW_CASES])
def test_pw_gemm_pyramid_layers(ops, case, launches):
    """ops.conv2d(dxe, wed, Cin, 1, residual=dy on skip blocks, w_tc=tc_packs(We)[1]) as MBConvFn.backward calls it on
    the fp32 route, and the NB 2 expand forward with three images per m-tile, into a NaN-filled guarded output, against
    a float64 matmul plus the residual: whole tensor, each image, each 64-column block.  Controls: the last column block
    without its last k-block, hi*hi only, the output without the residual"""
    s = _pwg_setup(ops, case)
    B, H, W, Cin, Cout, M = (s[k] for k in ('B', 'H', 'W', 'Cin', 'Cout', 'M'))
    y, outs = s['launch']()
    operand = s['x'].view(M, Cin).double()
    prod = operand @ s['weight'].t()
    want = prod + (s['res'].double().view(M, Cout) if s['res'] is not None else 0.0)
    got = y.view(M, Cout)
    plan = _pwg_plan(B, H, W, Cin, Cout, False, _sms())
    what = '%s block %d %s %d->%d B=%d %dx%d%s: KB %d, BN %d x %d n-tiles, %s weights, NS %d, %d units per CTA, ' \
           '%d images per tile' % (case[0], case[1], case[2], Cin, Cout, B, H, W, ' + residual' if s['res'] is not None
                                   else '', plan['KB'], plan['BN'], plan['ntn'], 'resident' if plan['bres'] else
                                   'streamed', plan['NS'], plan['upc'], plan['images'])
    print(what)
    _check_launch(launches[str(case)], 'pw_gemm_kernel<%d>(' % plan['NB'], plan['grid'], 'pw_gemm', plan['smem'])
    assert torch.isfinite(got).all(), (what, 'NaN or inf in the output')
    _check_guards(outs, what)
    e, img, blk = _pw_errs(got, want, B)
    print('  rel err %.2e (bound %.0e), worst image %.2e, worst 64-column block %.2e (bound %.0e)'
          % (e, TOL_TC, img, blk, TOL_ROW))
    assert e < TOL_TC and img < TOL_ROW and blk < TOL_ROW, (what, e, img, blk)
    k0, n0 = 64 * (plan['KB'] - 1), (Cout - 1) // 64 * 64
    miss = want.clone()
    miss[:, n0:] -= operand[:, k0:] @ s['weight'][n0:, k0:].t()
    ctrl_k = _pw_errs(got, miss, B)[2]
    ctrl_hh = _rel(operand.to(torch.bfloat16).double() @ s['weight'].to(torch.bfloat16).double().t(), prod)
    msg = '  controls: last column block without its last k-block %.2e, hi*hi only %.2e' % (ctrl_k, ctrl_hh)
    assert ctrl_k > TOL_ROW and ctrl_hh > TOL_TC, (ctrl_k, ctrl_hh)
    if s['res'] is not None:
        ctrl_res = _rel(got, prod)
        msg += ', without the residual %.2e' % ctrl_res
        assert ctrl_res > TOL_TC, ctrl_res
    print(msg)


# ------------------------------------------------------------------------------------------------
# 2. pw_wgrad_kernel with dy in fp32, and the NB 2 instances
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', WGRAD_CASES, ids=['%s-%d-%s-B%d' % c for c in WGRAD_CASES])
def test_pw_wgrad_pyramid_layers(ops, case, launches):
    """dW += dy^T act(x) as MBConvFn.backward calls it (plain: conv_wgrad(x, dxe, dWe) with dy in fp32), accumulated into
    a non-zero dw with a zero guard after it, against float64 image by image: whole tensor and each output-channel row.
    Control: the reference without the pixels one CTA accumulates"""
    s = _wgrad_setup(ops, case)
    B, H, W, Cin, Cout, dy, act = (s[k] for k in ('B', 'H', 'W', 'Cin', 'Cout', 'dy', 'act'))
    plan = _pw_plan(B, H, W, Cin, Cout, _sms())
    ref = torch.zeros(Cout, Cin, dtype=torch.float64, device=_dev())
    for b in range(B):
        ref += dy[b].reshape(-1, Cout).double().t() @ act(b)
    npx = min(plan['pixels'], H * W)
    first = dy[0].reshape(-1, Cout)[:npx].double().t() @ act(0, slice(0, npx))
    dw = _Out((Cout, Cin, 1, 1), 0.0)
    dw0 = _randn(s['g'], Cout, Cin, 1, 1) * float(ref.std())
    dw.t.copy_(dw0)
    s['launch'](dw.t)
    got = (dw.t.double() - dw0.double()).view(Cout, Cin)
    what = 'pw wgrad %s %s block %d %d->%d B=%d %dx%d: %d pixels per CTA (%d splits)' % (
        s['mode'], case[0], case[1], Cin, Cout, B, H, W, plan['pixels'], plan['splits'])
    print(what)
    _check_launch(launches[str(case)], 'pw_wgrad_kernel<%d>(' % plan['NB'], plan['grid'], 'pw_wgrad')
    _check_guards([dw], what)

    def errs(want):
        return _rel(got, want), float(((got - want).norm(dim=1) / want.norm(dim=1)).max())
    e, row = errs(ref)
    ctrl, ctrl_row = errs(ref - first)
    print('  rel err %.2e (bound %.0e), worst row %.2e (bound %.0e); control without %d pixels %.2e / %.2e'
          % (e, TOL_TC, row, TOL_ROW, npx, ctrl, ctrl_row))
    assert e < TOL_TC and row < TOL_ROW, (e, row)
    assert ctrl > TOL_TC and ctrl_row > TOL_ROW, (ctrl, ctrl_row)


# ------------------------------------------------------------------------------------------------
# 3. depthwise forward and backward with a partial last channel group
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', DW_CASES, ids=['%s-%d-B%d' % c for c in DW_CASES])
def test_dwconv_partial_channel_group(case, launches):
    """z1, each image's SE mean, dx, each tap of dW and both BN affine gradients at C % 16 != 0, native maps and
    tile-per-CTA plans, against float64 autograd image by image; the same on the last (partial) 16-channel group alone;
    nothing lands in the guard after any output.  Controls: image 0's mean without one forward tile, dW without the
    output gradient of one backward tile"""
    s = _dw_setup(case)
    k, st, pre, C, H, W, B, Ho, Wo = (s[n] for n in ('k', 's', 'pre', 'C', 'H', 'W', 'B', 'Ho', 'Wo'))
    x, wd, bn, gate, dq, dmean, o = (s[n] for n in ('x', 'wd', 'bn', 'gate', 'dq', 'dmean', 'out'))
    s['fwd']()
    s['bwd']()
    torch.cuda.synchronize()
    c0 = C // 16 * 16                               # the last channel group: C - c0 real channels of 16
    sq = {n: [0.0, 0.0] for n in ('z1', 'dx', 'z1_last', 'dx_last')}
    mean_ref = torch.zeros(B, C, dtype=torch.float64, device=_dev())
    dw_ref = torch.zeros(C, 1, k, k, dtype=torch.float64, device=_dev())
    bn_ref = None
    for b in range(B):
        z_r, m_r, dx_r, dw_r, bg_r = _dw_reference(x[b], wd, bn, gate[b], dq[b], dmean[b], k, st, pre)
        for n, got, want in (('z1', o['z1'].t[b], z_r), ('dx', o['dx'].t[b], dx_r)):
            sq[n][0] += float((got.double() - want).norm()) ** 2
            sq[n][1] += float(want.norm()) ** 2
            sq[n + '_last'][0] += float((got[..., c0:].double() - want[..., c0:]).norm()) ** 2
            sq[n + '_last'][1] += float(want[..., c0:].norm()) ** 2
        mean_ref[b] = m_r
        dw_ref += dw_r
        bn_ref = bg_r if bn_ref is None else [a + c for a, c in zip(bn_ref, bg_r)]
    got_dw = o['dw'].t.double().view(C, -1)
    want_dw = dw_ref.view(C, -1)
    errs = {n: (a / w) ** 0.5 for n, (a, w) in sq.items()}
    errs.update(mean_rows=max(_rel(o['mean'].t[b], mean_ref[b]) for b in range(B)),
                mean_last=max(_rel(o['mean'].t[b, c0:], mean_ref[b, c0:]) for b in range(B)),
                dw=_rel(got_dw, want_dw), dw_taps=max(_rel(got_dw[:, t], want_dw[:, t]) for t in range(k * k)),
                dw_last=_rel(got_dw[c0:], want_dw[c0:]))
    names = ['dgamma1', 'dbeta1', 'dgamma0', 'dbeta0'][:len(bn_ref)]
    for n, want in zip(names, bn_ref):
        errs[n] = _rel(o[n].t, want)
        errs[n + '_last'] = _rel(o[n].t[c0:], want[c0:])
    fp = _dw_plan('fwd', k, st, C, H, W, B)
    bp = _dw_plan('bwd', k, st, C, H, W, B)
    what = 'dw %s block %d k%d s%d BN0=%s C=%d (last group %d of 16 channels) %dx%d B=%d: fwd %d tiles per CTA (of ' \
           '%d), bwd %d (of %d)' % (case[0], case[1], k, st, pre, C, C - c0, H, W, B, fp['tpc'], fp['ntiles'],
                                    bp['tpc'], bp['ntiles'])
    print(what)
    tmpl = '%d,%d,%s,%s>' % (k, st, str(pre).lower(), '%s')
    _check_launch(launches[str(case) + ' fwd'], 'dw_fwd_fused_kernel<' + tmpl % str(fp['small']).lower(), fp['grid'],
                  'forward')
    _check_launch(launches[str(case) + ' bwd'], 'dw_bwd_fused_kernel<' + tmpl % str(bp['small']).lower(), bp['grid'],
                  'backward')
    _check_guards(list(o.values()), what)
    print('  %s (bound %.0e)' % (', '.join('%s %.2e' % kv for kv in errs.items()), TOL_DW))
    # controls: image 0's mean without the first forward tile; dW without the output gradient of the first backward tile
    ty, tx = fp['tile']
    z_r, _, _, dw_full0, _ = _dw_reference(x[0], wd, bn, gate[0], dq[0], dmean[0], k, st, pre)
    a1 = _swish(z_r * s['sc1'].double() + s['sh1'].double())
    ctrl_mean = _rel(o['mean'].t[0], mean_ref[0] - a1[:ty, :tx].sum(dim=(0, 1)) / (Ho * Wo))
    mask = torch.ones(Ho, Wo, dtype=torch.float64, device=_dev())
    cy, cx = bp['tile']
    mask[:cy, :cx] = 0
    dw_drop0 = _dw_reference(x[0], wd, bn, gate[0], dq[0], dmean[0], k, st, pre, mask=mask)[3]
    want_ctrl = (dw_ref - dw_full0 + dw_drop0).view(C, -1)
    ctrl_tap = max(_rel(got_dw[:, t], want_ctrl[:, t]) for t in range(k * k))
    print('  controls: mean without a tile %.2e, dW without a tile %.2e' % (ctrl_mean, ctrl_tap))
    assert max(errs.values()) < TOL_DW, errs
    assert ctrl_mean > TOL_DW and ctrl_tap > TOL_DW, (ctrl_mean, ctrl_tap)


# ------------------------------------------------------------------------------------------------
# 4. the stem at native sizes
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', STEM_CASES, ids=['%s-B%d' % c for c in STEM_CASES])
def test_stem_native_sizes(case, launches):
    """effdet_stem_fwd (z and y), effdet_bnact_bwd in SWISH mode and effdet_stem_wgrad into guarded buffers, against
    F.pad(x, (0, 1, 0, 1)), a stride-2 conv and BN + swish in float64 on the device, four images at a time; control: dW
    without the last 64-pixel row segment"""
    s = _stem_setup(case)
    C0, H, W, B, Ho, Wo, x, w, o = (s[n] for n in ('C0', 'H', 'W', 'B', 'Ho', 'Wo', 'x', 'w', 'out'))
    s['fwd']()
    s['bnact']()
    s['wgrad']()
    sq = {n: [0.0, 0.0] for n in ('z', 'y', 'dz')}
    dw_ref = torch.zeros(C0, 3, 3, 3, dtype=torch.float64, device=_dev())
    dg_ref = torch.zeros(C0, dtype=torch.float64, device=_dev())
    db_ref = torch.zeros_like(dg_ref)
    G = 4
    for b0 in range(0, B, G):
        sl = slice(b0, min(B, b0 + G))
        xp = F.pad(x[sl].double(), (0, 1, 0, 1))
        wr = w.double().requires_grad_(True)
        gr, br = s['gamma'].double().requires_grad_(True), s['beta'].double().requires_grad_(True)
        zr = F.conv2d(xp, wr, None, 2)
        zr.retain_grad()
        u = (zr - s['mu'].double()[:, None, None]) / torch.sqrt(s['var'].double()[:, None, None] + BN_EPS) * \
            gr[:, None, None] + br[:, None, None]
        yr = _swish(u)
        (yr * s['dy'][sl].permute(0, 3, 1, 2).double()).sum().backward()
        for n, want in (('z', zr), ('y', yr), ('dz', zr.grad)):
            want = want.detach().permute(0, 2, 3, 1)
            sq[n][0] += float((o[n].t[sl].double() - want).norm()) ** 2
            sq[n][1] += float(want.norm()) ** 2
        dw_ref += wr.grad
        dg_ref += gr.grad
        db_ref += br.grad
        if b0 + G >= B:                 # control: the last row segment of the last image
            seg = torch.zeros_like(zr.grad[-1:])
            ox0 = (Wo - 1) // 64 * 64
            seg[..., -1, ox0:] = zr.grad[-1:, :, -1, ox0:]
            last_seg = torch.nn.grad.conv2d_weight(xp[-1:], w.shape, seg, 2)
        del xp, zr, u, yr
    plan = _stem_plan(B, H, W, C0, _sms())
    errs = {n: (a / b) ** 0.5 for n, (a, b) in sq.items()}
    sums = dict(dw=_rel(o['dw'].t, dw_ref), dgamma=_rel(o['dgamma'].t, dg_ref), dbeta=_rel(o['dbeta'].t, db_ref))
    ctrl = _rel(o['dw'].t, dw_ref - last_seg)
    what = 'stem %s C0=%d %dx%d B=%d: TPG %d, %d segments per CTA' % (case[0], C0, H, W, B, plan['tpg'],
                                                                      plan['segs_per_cta'])
    print(what)
    _check_launch(launches[str(case)], 'stem_wgrad_kernel<%d>(' % plan['tpg'], plan['grid'], 'stem_wgrad')
    _check_guards(list(o.values()), what)
    print('  %s (bound %.0e); %s (bound %.0e); control without the last segment %.2e'
          % (', '.join('%s %.2e' % kv for kv in errs.items()), TOL_EXACT,
             ', '.join('%s %.2e' % kv for kv in sums.items()), TOL_SUM, ctrl))
    assert max(errs.values()) < TOL_EXACT, errs
    assert max(sums.values()) < TOL_SUM, sums
    assert ctrl > TOL_SUM, ctrl


# ------------------------------------------------------------------------------------------------
# 5. MBConvFn composed on the fp32 route
# ------------------------------------------------------------------------------------------------

def _block_params(cfg, i):
    """random parameters of backbone block i, drawn as tests/test_pointwise_se_parity.py draws them"""
    q = 'backbone._blocks.%d.' % i
    g = torch.Generator().manual_seed(1000 + i)
    sd = {}
    for n, shape, kind in O.state_dict_spec(cfg):
        if not n.startswith(q) or kind == 'bn_n':
            continue
        if kind == 'conv':
            t = torch.randn(shape, generator=g) * (1.5 / (shape[1] * shape[2] * shape[3]) ** 0.5)
        elif kind == 'bn_w':
            t = torch.rand(shape, generator=g) * 0.6 + 0.7
        elif kind == 'bn_rv':
            t = torch.rand(shape, generator=g) + 0.6
        else:
            t = torch.randn(shape, generator=g) * 0.2
        sd[n] = t.to(_dev())
    return q, sd


@pytest.mark.gpu
@pytest.mark.parametrize('geo,block,B,drop', MB_CASES, ids=['%s-%d-B%d-%s' % c for c in MB_CASES])
def test_mbconv_block_fp32_route(ops, geo, block, B, drop):
    """MBConvFn forward and backward at a block whose map has no pixel box (planes_ok false: dxe in fp32, conv_wgrad
    and conv2d with residual=dy on a skip block) against float64 autograd of O.mbconv_forward: output, input gradient,
    every parameter gradient.  Controls: the input gradient against a reference with a bf16-rounded expand weight, and
    on the skip block without the skip path's dy"""
    net, size = PYRAMIDS[geo]
    cfg = O.make_config(net)
    blk = cfg['blocks'][block]
    c = _find(geo, block, B, 'pw', route='expand_fwd')
    H, W = c['shape'][1:3]
    assert not ops.planes_ok(B, H, W, blk['cin'] * blk['e']) and blk['skip'] == drop
    q, sd = _block_params(cfg, block)
    g = _gen(77 + block)
    x = _randn(g, B, H, W, blk['cin'])
    k, s = blk['k'], blk['s']
    left, right, top, bottom = O.same_pad(k, s, cfg['nominal'])
    kcfg = dict(k=k, s=s, eps=O.BN_EPS, expand=True, skip=blk['skip'], pad_t=top, pad_l=left, pad_h=top + bottom,
                pad_w=left + right)
    keep = None
    if drop:                    # drop_connect_scale's floor(kp + u) / kp, with image 0 dropped and image 1 kept
        kp = 1 - O.DROP_CONNECT_RATE * block / len(cfg['blocks'])
        keep = torch.floor(kp + _rand(g, B)) / kp
        keep[0], keep[1] = 0.0, 1.0 / kp
    names = [q + '_expand_conv.weight'] + [q + '_bn0.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
    names += [q + '_depthwise_conv.weight'] + [q + '_bn1.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
    names += [q + '_se_reduce.weight', q + '_se_reduce.bias', q + '_se_expand.weight', q + '_se_expand.bias',
              q + '_project_conv.weight'] + [q + '_bn2.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
    params = [sd[n].clone().requires_grad_('running' not in n) for n in names]
    xg = x.clone().requires_grad_(True)
    y = ops.MBConvFn.apply(xg, keep, kcfg, *params)
    dy = _randn(g, *y.shape)
    y.backward(dy)

    def reference(sd_):
        sd64 = {n: v.double().requires_grad_('running' not in n) for n, v in sd_.items()}
        x64 = x.permute(0, 3, 1, 2).double().requires_grad_(True)
        y64 = O.mbconv_forward(sd64, q, blk, x64, cfg['nominal'])
        if keep is not None:
            y64 = (y64 - x64) * keep.double().view(B, 1, 1, 1) + x64
        y64.backward(dy.permute(0, 3, 1, 2).double())
        return y64.detach(), x64.grad, sd64
    y64, dx64, sd64 = reference(sd)
    dx = xg.grad.permute(0, 3, 1, 2)
    errs = {'y': _rel(y.detach().permute(0, 3, 1, 2), y64), 'dx': _rel(dx, dx64)}
    for n, p in zip(names, params):
        if p.requires_grad:
            errs[n[len(q):]] = _rel(p.grad, sd64[n].grad)
    print('mbconv %s block %d (B %d, %dx%d, %d->%d, expand %d, skip %s, drop-connect %s): %s (bounds %.0e / %.0e)'
          % (geo, block, B, H, W, blk['cin'], blk['cout'], blk['cin'] * blk['e'], blk['skip'], drop,
             ', '.join('%s %.2e' % kv for kv in errs.items()), TOL_MB_FWD, TOL_MB_GRAD))
    assert errs['y'] < TOL_MB_FWD, errs
    assert max(v for n, v in errs.items() if n != 'y') < TOL_MB_GRAD, errs
    we = q + '_expand_conv.weight'
    ctrl = dict(bf16_expand_weight=_rel(dx, reference(dict(sd, **{we: sd[we].to(torch.bfloat16).float()}))[1]))
    if blk['skip']:
        ctrl['without_dy'] = _rel(dx - dy.permute(0, 3, 1, 2), dx64)
    print('  controls: %s' % ', '.join('%s %.2e' % kv for kv in ctrl.items()))
    assert min(ctrl.values()) > TOL_MB_GRAD, ctrl


# ------------------------------------------------------------------------------------------------
# 6. the SE gate and spatial_reduce_act at the pyramids' shapes
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('C,S', list(_se_cases(_walk_all())))
def test_se_gate_at_pyramids(C, S):
    """tests/test_pointwise_se_parity.py's SE gate check (float64 autograd, bit-identical backward calls, controls) at
    every B of the walk with this (C, S) that the benchmark's shapes do not have"""
    for B in _se_cases(_walk_all())[(C, S)]:
        _se_gate_check(B, C, S)


@pytest.mark.gpu
@pytest.mark.parametrize('B,HW,C', _sra_pyramid_cases(_walk_all()))
def test_spatial_reduce_act_at_pyramids(B, HW, C, launches):
    """tests/test_pointwise_se_parity.py's spatial_reduce_act check (float64 per image, grid against _row_grid, control
    without one row block) at the walk's most rows per block and most channel chunks"""
    _sra_check(B, HW, C, launches)
