"""Kernel-level fp64 parity of the MBConv block's pointwise GEMM and squeeze-excite gate at the benchmark's launch plans.

  pw_gemm_kernel       every 1x1 conv of the backbone and the BiFPN laterals (pw_gemm.cu): the expand and project
                       forwards, both data gradients, the lateral forward and data gradient
  se_squeeze_kernel, se_excite_kernel, se_bwd_dp_kernel, se_bwd_dmean_kernel, se_bwd_dw_kernel   the squeeze-excite gate
                       and its backward (se_ops.cu)
  spatial_reduce_kernel the SE backward's dgate = sum over pixels of dq * swish(BN1(z1)) (mbconv_ops.cu)

pw_gemm_launch picks its plan from the problem size: the n-tile width BN (pw_gemm_kernel<1> or <2>), the k-block count
KB, resident or streamed weights (bres), the ring depth NS, one or two fp32 half-boxes per stage, and a grid of
min(units, SMs) persistent CTAs.  When a 128-row m-tile holds rows of several images (maps of 8x8 and 4x4 at d0 512^2),
the converter warps read the SE gate row by row and the epilogue finds each row's image.  This file

  * mirrors pw_gemm_launch (_pwg_plan) and mbconv_ops.cu's row_grid (_row_grid), walks every pw_gemm call, SE gate and
    spatial_reduce_act of bench.CONFIGS (_bench_calls) and checks, without a GPU, that the cases below reach every
    (route, NB, bres, half-boxes, NS, images per tile) class the benchmark reaches, and its longest K (KB 54), most
    n-tiles (27) and most units per CTA (125) (test_cases_reach_benchmark_plans);
  * holds each pw_gemm call, entered through ops.conv2d / ops.conv2d_from_planes with the arguments MBConvFn and the
    laterals pass, into NaN-filled outputs, to the prologue'd operand times the weight as a float64 matmul on the device:
    the whole tensor, each image and each 64-column block;
  * holds the SE gate to float64 autograd of sigmoid(W2 swish(W1 mean + b1) + b2) at every (B, C, S) of the walk, plus
    C = 16 384 (the shared-memory opt-in of se_bwd_dp_kernel) and C not a multiple of 128, and two backward calls to
    bit-identical results (the kernels have no atomics);
  * holds spatial_reduce_act to float64 at the benchmark's largest shapes;
  * runs MBConvFn forward and backward at d0 blocks 1, 12 and 15 and a d4 skip block with drop-connect against float64
    autograd of O.mbconv_forward: the wiring between the kernels (which mean, s_pre and gate reach which kernel);
  * records every launch once under torch.profiler in a fresh interpreter (the launches fixture) and compares kernel
    name, grid and dynamic shared memory with the mirrors.

Bounds (norm-relative error ||got - want|| / ||want||):
  TOL_TC    = 3e-5  a whole bf16x3 output tensor
  TOL_ROW   = 1e-4  each image and each 64-column block of it
  TOL_EXACT = 5e-6  the exact-fp32 SE outputs, per image (s_pre, gate, dmean) and per row (dW1, dW2), db1, db2
  TOL_SUM   = 2e-5  spatial_reduce_act (sums built from atomics), per image
  TOL_MB_FWD = 1e-4, TOL_MB_GRAD = 2e-4  the composed block: output, and the input and every parameter gradient
Negative controls, each of which must exceed the bound it targets: the neighbouring image's gate on the second image's
rows of a shared tile (per image); one 64-column block whose reference lacks its last k-block (per block); hi*hi bf16
products only (whole tensor); the SE reference from the wrong image's mean (s_pre per image); dW2 without the last
image (per row); dp2 without the (1 - g) factor (db2); spatial_reduce_act without one row block (per image).

Measured on an H100 80GB HBM3 at 700 W (worst case of each test):
  pw_gemm_kernel, every layer but the longest K   whole tensor 3.2e-6 .. 6.0e-6, worst image 6.7e-6 and worst 64-column
                                                  block 6.0e-6 (the project forward of d0 blocks 12 and 15, 2 and 8
                                                  images per m-tile)
  pw_gemm_kernel, d7 3456 -> 576 (KB = 54)        1.33e-5 whole, 1.36e-5 worst 64-column block: 44 % of TOL_TC.  The
                                                  error grows with K (about 4.5e-6 at KB <= 9); the gather path's
                                                  3.2e-9 per term predicted 1.1e-5 here.  No change to the kernel.
  SE gate, every (B, C, S)                        s_pre 4.6e-7, gate 1.3e-7, dp2 8.8e-8, dp1 9.0e-7, dmean 9.0e-7 (per
                                                  image); dW1 8.6e-7, dW2 4.4e-7 (whole); their rows 1.8e-7, 4.0e-7;
                                                  db1 9.0e-7, db2 1.4e-7.  The worst at C = 16 384.
  spatial_reduce_act                              3.3e-7 per image
  MBConvFn composed                               output 7.2e-6, input gradient 9.5e-6, parameter gradients 1.65e-5
                                                  (expand and project weights, the bf16x3 weight gradients)
The weakest controls: the last k-block missing from one column block 1.2e-1, hi*hi only 2.3e-3, the neighbouring
image's gate 7.9e-1, the wrong image's mean 8.7e-1, dW2 without the last image 7.8e-1, dp2 without (1 - g) 5.2e-1,
spatial_reduce_act without one row block 7.6e-2."""
import json
import os
import pathlib
import subprocess
import sys
from collections import Counter

import pytest
import torch

import effdet_oracle as O
from test_benchmark_plans import SMS, TOL_EXACT, TOL_ROW, TOL_SUM, TOL_TC, _dw_out, _stem_out
from test_planes_path_parity import _box
from test_planes_path_parity import ops  # noqa: F401  (the bf16x3 fixture)

TOL_MB_FWD = 1e-4
TOL_MB_GRAD = 2e-4

# pw_gemm.cu / tc_ptx.cuh constants of the launcher's shared-memory plan
PW_MAX_STAGES = 6                     # kPwMaxStages
PW_A32_HALF = 128 * 128               # kPwA32Half: one fp32 half-box, 128 rows x 32 floats
PW_A16 = 2 * 128 * 128                # kPwA16: one bf16 hi + lo stage, 128 rows x 64 bf16 each
PW_FIXED = 64 * 68 * 4 + 512 + 3 * 128 * 4 + 1024   # kRowsBytes + kPwBarBytes + kPwChanBytes + alignment slack
PW_SMEM = 227 * 1024
PW_BRES_MAX = 64 * 1024               # weights resident when every tile of the layer fits here


def _cdiv(a, b):
    return -(-a // b)


def _dev():
    return torch.device('cuda:0')


# ------------------------------------------------------------------------------------------------
# mirrors of pw_gemm_launch (pw_gemm.cu) and row_grid (mbconv_ops.cu)
# ------------------------------------------------------------------------------------------------

def _images_per_tile(B, HW):
    """the largest number of images whose rows share one 128-row m-tile (rows below M only)"""
    inside = Counter((b * HW) // 128 for b in range(1, B) if (b * HW) % 128)
    return 1 + max(inside.values(), default=0)


def _pwg_plan(B, H, W, Cin, Cout, planes, sms):
    """one pw_gemm_launch: KB, BN, ntn, units, half-boxes (None in planes mode), bres, NS, dynamic shared memory bytes,
    grid, units per CTA, the template NB and the most images in one m-tile"""
    M = B * H * W
    KB = _cdiv(Cin, 64)
    ntn = _cdiv(Cout, 128)
    BN = _cdiv(_cdiv(Cout, ntn), 64) * 64
    ntn = _cdiv(Cout, BN)
    units = _cdiv(M, 128) * ntn
    halves = 2 if Cin > 32 else 1
    a_stage = PW_A16 if planes else halves * PW_A32_HALF
    b_all = ntn * KB * BN * 256
    bres = b_all <= PW_BRES_MAX
    stage = a_stage + (0 if bres else BN * 256)
    fixed = (0 if planes else 2 * PW_A16) + PW_FIXED + (b_all if bres else 0)
    NS = min((PW_SMEM - fixed) // stage, PW_MAX_STAGES)
    assert NS >= 2, ('the launcher refuses', B, H, W, Cin, Cout)
    grid = min(units, sms)
    return dict(KB=KB, BN=BN, ntn=ntn, units=units, halves=None if planes else halves, bres=bres, NS=NS,
                smem=fixed + NS * stage, grid=(grid, 1, 1), upc=_cdiv(units, grid), NB=BN // 64,
                images=_images_per_tile(B, H * W))


def _row_grid(HW, cvecs, B, sms):
    """(grid, rows per block) of row_grid for C / 4 = cvecs channel vectors"""
    rows = 1 if cvecs >= 256 else 256 // cvecs
    chunks = 1 if cvecs <= 256 else _cdiv(cvecs, 256)
    want = max(1, (sms * 4 + B * chunks - 1) // (B * chunks))
    rpb = max(_cdiv(HW, want), rows * 8)
    return (_cdiv(HW, rpb), chunks, B), rpb


def _pw_class(route, p):
    return (route, p['NB'], p['bres'], p['halves'], p['NS'], min(p['images'], 3))


# ------------------------------------------------------------------------------------------------
# the benchmark's calls
# ------------------------------------------------------------------------------------------------

ROUTES = ('expand_fwd', 'project_fwd', 'project_dgrad', 'expand_dgrad_planes', 'expand_dgrad_fp32', 'lateral_fwd',
          'lateral_dgrad')


def _bench_calls(name):
    """every pw_gemm call MBConvFn and the BiFPN laterals make in one step of bench.CONFIGS[name] (forward and backward
    for the train configs), every SE gate (B, C, S) and every spatial_reduce_act (B, HW, C).  A pw call is a dict of
    config, block (an int, or 'lateral<i>'), route, shape (B, H, W, Cin, Cout) and skip"""
    from bench import CONFIGS
    c = CONFIGS[name]
    cfg = O.make_config(c['net'], num_classes=c['K'], W_bifpn=c['W'], D_bifpn=c['D'])
    B, train = c['bs'], c['mode'] == 'train'
    H, W = _stem_out(c['size'], c['size'])
    pw, se, sra, feats = [], [], [], []

    def add(block, route, h, w, cin, cout, skip=False):
        pw.append(dict(config=name, block=block, route=route, shape=(B, h, w, cin, cout), skip=skip))
    for i, blk in enumerate(cfg['blocks']):
        mid = blk['cin'] * blk['e']
        expand = blk['e'] != 1
        Ho, Wo = _dw_out(blk['k'], blk['s'], H, W)
        if expand:
            add(i, 'expand_fwd', H, W, blk['cin'], mid)
        add(i, 'project_fwd', Ho, Wo, mid, blk['cout'], blk['skip'])
        se.append((B, mid, blk['sq']))
        if train:
            add(i, 'project_dgrad', Ho, Wo, blk['cout'], mid)
            sra.append((B, Ho * Wo, mid))
            if expand:       # MBConvFn.backward: planes when ops.planes_ok(B, H, W, mid)
                planes = mid % 8 == 0 and _box(B, H, W) is not None
                add(i, 'expand_dgrad_planes' if planes else 'expand_dgrad_fp32', H, W, mid, blk['cin'], blk['skip'])
        H, W = Ho, Wo
        if i in cfg['stage_last']:
            feats.append((H, W, blk['cout']))
    for i, (h, w, ch) in enumerate(feats[-5:]):
        add('lateral%d' % i, 'lateral_fwd', h, w, ch, cfg['W'])
        if train:
            add('lateral%d' % i, 'lateral_dgrad', h, w, cfg['W'], ch)
    return pw, se, sra


def _find(config, block, route):
    calls = [c for c in _bench_calls(config)[0] if c['block'] == block and c['route'] == route]
    assert len(calls) == 1, (config, block, route, calls)
    return calls[0]


def _plan_of(call, sms=SMS):
    return _pwg_plan(*call['shape'], call['route'] == 'expand_dgrad_planes', sms)


# ------------------------------------------------------------------------------------------------
# the GPU cases
# ------------------------------------------------------------------------------------------------

# pw_gemm: (config, block, route), each at the benchmark's own B, H, W, Cin and Cout
PW_CASES = [
    ('d0', 0, 'project_fwd'), ('d0', 0, 'project_dgrad'),
    ('d0', 1, 'expand_fwd'), ('d0', 1, 'project_fwd'), ('d0', 1, 'project_dgrad'), ('d0', 1, 'expand_dgrad_planes'),
    ('d0', 2, 'project_fwd'), ('d0', 4, 'expand_fwd'), ('d0', 4, 'project_dgrad'),
    ('d0', 6, 'expand_fwd'), ('d0', 6, 'project_dgrad'), ('d0', 6, 'expand_dgrad_planes'),
    ('d0', 12, 'expand_fwd'), ('d0', 12, 'project_fwd'), ('d0', 12, 'project_dgrad'),
    ('d0', 12, 'expand_dgrad_planes'),
    ('d0', 15, 'expand_fwd'), ('d0', 15, 'project_fwd'), ('d0', 15, 'project_dgrad'),
    ('d0', 15, 'expand_dgrad_planes'),
    ('d0', 'lateral0', 'lateral_fwd'), ('d0', 'lateral0', 'lateral_dgrad'), ('d0', 'lateral1', 'lateral_dgrad'),
    ('d0', 'lateral3', 'lateral_fwd'), ('d0', 'lateral3', 'lateral_dgrad'),
    ('d0', 'lateral4', 'lateral_fwd'), ('d0', 'lateral4', 'lateral_dgrad'),
    ('d4', 0, 'project_fwd'), ('d4', 1, 'project_fwd'), ('d4', 1, 'project_dgrad'),
    ('d4', 2, 'expand_fwd'), ('d4', 2, 'project_dgrad'), ('d4', 2, 'expand_dgrad_planes'),
    ('d4', 7, 'project_fwd'), ('d4', 7, 'expand_dgrad_planes'),
    ('d4', 'lateral0', 'lateral_fwd'), ('d4', 'lateral0', 'lateral_dgrad'),
    ('d4', 'lateral1', 'lateral_fwd'), ('d4', 'lateral1', 'lateral_dgrad'),
    ('d4', 'lateral4', 'lateral_fwd'), ('d4', 'lateral4', 'lateral_dgrad'),
    ('d7', 'last', 'expand_fwd'), ('d7', 'last', 'project_fwd'),
]

# the SE gate: every distinct (B, C, S) of the walk, plus the shared-memory opt-in and channel counts off the tiles
SE_EXTRA = [(2, 16384, 64), (3, 1000, 37), (5, 130, 9)]
# spatial_reduce_act: the benchmark's largest (B, HW, C) of each train config, and the smallest map of d0
SRA_CONFIGS = ('d0', 'd4')
# the composed block: (config, block, drop-connect)
MB_CASES = [('d0', 1, False), ('d0', 12, True), ('d0', 15, False), ('d4', 'skip', True)]


def _resolve_block(config, block):
    """'last': the last block; 'skip': the first skip block with an expand conv"""
    from bench import CONFIGS
    c = CONFIGS[config]
    blocks = O.make_config(c['net'], num_classes=c['K'], W_bifpn=c['W'], D_bifpn=c['D'])['blocks']
    if block == 'last':
        return len(blocks) - 1
    if block == 'skip':
        return next(i for i, b in enumerate(blocks) if b['skip'] and b['e'] != 1)
    return block


def _case_call(case):
    config, block, route = case
    if not (isinstance(block, str) and block.startswith('lateral')):
        block = _resolve_block(config, block)
    return _find(config, block, route)


def _se_shapes():
    shapes = set()
    for name in ('d0', 'd4', 'd7'):
        shapes |= set(_bench_calls(name)[1])
    return sorted(shapes) + SE_EXTRA


def _sra_cases():
    out = []
    for name in SRA_CONFIGS:
        sra = _bench_calls(name)[2]
        out.append(max(sra, key=lambda t: t[0] * t[1] * t[2]))
        if name == 'd0':
            out.append(min(sra, key=lambda t: t[1]))
    return out


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_mirrors():
    """the launchers' arithmetic on the figures that motivated the cases (132 SMs)"""
    p = _pwg_plan(32, 256, 256, 32, 16, False, SMS)            # d0 block 0 project: 16 384 m-tiles on 132 CTAs
    assert (p['units'], p['upc'], p['grid'], p['NB'], p['halves'], p['bres']) == (16384, 125, (132, 1, 1), 1, 1, True)
    p = _pwg_plan(1, 12, 12, 3456, 576, False, SMS)            # d7's last project: the longest K
    assert (p['KB'], p['BN'], p['ntn'], p['bres'], p['units']) == (54, 128, 5, False, 10)
    p = _pwg_plan(1, 12, 12, 576, 3456, False, SMS)            # ... and its expand: the most n-tiles
    assert (p['ntn'], p['BN'], p['KB']) == (27, 128, 9)
    assert _images_per_tile(32, 16) == 8 and _images_per_tile(32, 64) == 2 and _images_per_tile(32, 4096) == 1
    assert _images_per_tile(3, 100) == 2 and _images_per_tile(1, 16) == 1
    assert _row_grid(16384, 24, 32, SMS) == ((17, 1, 32), 964)
    assert _row_grid(4, 288, 32, SMS) == ((1, 2, 32), 8)


def test_cases_reach_benchmark_plans():
    """every (route, NB, bres, half-boxes, NS, images-per-tile class) the benchmark reaches is reached by a GPU case, and
    the cases reach the benchmark's longest K, most n-tiles and most units per CTA; every SE and spatial_reduce_act
    shape of the walk is a case"""
    bench_cls, bench_plans = set(), []
    for name in ('d0', 'd4', 'd7'):
        for c in _bench_calls(name)[0]:
            p = _plan_of(c)
            bench_cls.add(_pw_class(c['route'], p))
            bench_plans.append(p)
    case_plans = [(case, _plan_of(_case_call(case))) for case in PW_CASES]
    case_cls = {_pw_class(case[2], p) for case, p in case_plans}
    assert bench_cls <= case_cls, sorted(bench_cls - case_cls, key=str)
    for key, want in (('KB', 54), ('ntn', 27), ('upc', 125)):
        assert max(p[key] for p in bench_plans) == want, key
        assert max(p[key] for _, p in case_plans) == want, key
    assert {r for r, *_ in bench_cls} == set(ROUTES) - {'expand_dgrad_fp32'}
    assert {min(p['images'], 3) for p in bench_plans} == {1, 2, 3}
    # the composed cases: one per images-per-tile class of the project forward, and a skip block with drop-connect
    imgs = set()
    for config, block, drop in MB_CASES:
        c = _find(config, _resolve_block(config, block), 'project_fwd')
        imgs.add(min(_plan_of(c)['images'], 3))
        assert not drop or c['skip']
    assert imgs == {1, 2, 3}
    se = {s for name in ('d0', 'd4', 'd7') for s in _bench_calls(name)[1]}
    assert se <= set(_se_shapes()) and any(C * 4 > 48 * 1024 for _, C, _ in _se_shapes())
    assert any(C % 128 for _, C, _ in _se_shapes()) and min(S for _, _, S in se) == 4


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


def _rel(got, want):
    """||got - want|| / ||want|| in float64 on the device; NaN anywhere in got gives NaN, which fails every bound"""
    n = float(want.norm())
    return float((got.double() - want).norm()) / n if n > 0 else float(float(got.double().norm()) > 0)


class _nan_outputs:
    """ops._empty hands out NaN-filled buffers inside the block: every output element a kernel leaves unwritten fails"""

    def __init__(self, ops):
        self.ops = ops

    def __enter__(self):
        self.old = self.ops._empty
        self.ops._empty = lambda shape, like: torch.full(shape, float('nan'), device=like.device, dtype=torch.float32)

    def __exit__(self, *exc):
        self.ops._empty = self.old


def _pw_errs(got, want, B):
    """(whole tensor, worst image, worst 64-column block) of [M, C] outputs with B images"""
    Cout = want.shape[1]
    per_img = max(_rel(a, b) for a, b in zip(got.view(B, -1, Cout), want.view(B, -1, Cout)))
    per_blk = max(_rel(got[:, n0:n0 + 64], want[:, n0:n0 + 64]) for n0 in range(0, Cout, 64))
    return _rel(got, want), per_img, per_blk


def _pw_setup(ops, case):
    """inputs, the pw_gemm call of `case` as MBConvFn / ConvBiasActFn make it, and the float64 reference:
    -> dict(launch, operand [M, Cin] float64, weight [Cout, Cin] float64, epilogue(prod) -> {output name: reference},
    outputs() -> {output name: [M, C] tensor})"""
    call = _case_call(case)
    route, (B, H, W, Cin, Cout), skip = call['route'], call['shape'], call['skip']
    M = B * H * W
    g = _gen(1 + PW_CASES.index(case))
    out = {}
    res = None
    if route in ('project_dgrad', 'expand_dgrad_planes', 'expand_dgrad_fp32', 'lateral_dgrad'):
        # the data gradient of the forward layer Cout -> Cin: the call runs Cin -> Cout on its dgrad pack
        w = _randn(g, Cin, Cout, 1, 1) * (1.5 / Cin ** 0.5)
        _, wd = ops.pack_conv(w)
        wtc = ops.tc_packs(w)[1]
        weight = w.view(Cin, Cout).t().double()
    else:
        w = _randn(g, Cout, Cin, 1, 1) * (1.5 / Cin ** 0.5)
        wf, _ = ops.pack_conv(w)
        wtc = ops.tc_packs(w)[0]
        weight = w.view(Cout, Cin).double()
    assert wtc is not None
    x = _randn(g, B, H, W, Cin)
    if skip:                                    # the project forward and expand data gradient of a skip block
        res = _randn(g, B, H, W, Cout)
    epi = dict()
    if route == 'expand_fwd':
        operand = x.view(M, Cin).double()

        def launch():
            out['y'] = ops.conv2d(x, wf, Cout, 1, w_tc=wtc)
    elif route == 'project_fwd':
        # z1 with a sprinkle of pre-activations out to about +-90, where fsigmoid's ex2.approx overflows
        big = _rand(g, B, H, W, Cin) < 0.004
        x = torch.where(big, (_rand(g, B, H, W, Cin) * 2 - 1) * 90, x * 2)
        sc1, sh1 = _rand(g, Cin) + 0.5, _randn(g, Cin) * 0.3
        gate = _rand(g, B, Cin)
        sc2, sh2 = _rand(g, Cout) + 0.5, _randn(g, Cout) * 0.3
        rs = None
        if skip:
            rs = torch.full((B,), 1.0 / 0.9, device=_dev())
            if B > 1:
                rs[B // 2] = 0.0                # one dropped image
        q = x.double() * sc1.double() + sh1.double()
        epi.update(q=q, gate=gate)
        operand = (_swish(q) * gate.double()[:, None, None, :]).view(M, Cin)
        epi['fn'] = lambda prod: dict(
            z=prod, y=((prod.view(B, -1, Cout) * sc2.double() + sh2.double())
                       * (rs.double()[:, None, None] if rs is not None else 1.0)
                       + (res.double().view(B, -1, Cout) if res is not None else 0.0)).view(M, Cout))

        def launch():
            out['y'], out['z'] = ops.conv2d(x, wf, Cout, 1, scale=sc2, shift=sh2, a_scale=gate, in_scale=sc1,
                                            in_shift=sh1, row_scale=rs, residual=res, save_z=True, w_tc=wtc)
    elif route == 'expand_dgrad_planes':
        hi = x.to(torch.bfloat16)
        planes = torch.stack([hi, (x - hi.float()).to(torch.bfloat16)]).contiguous()
        operand = (planes[0].double() + planes[1].double()).view(M, Cin)
        assert ops.planes_ok(B, H, W, Cin)

        def launch():
            y = torch.full((B, H, W, Cout), float('nan'), device=_dev())     # conv2d_from_planes, into a NaN buffer
            ops.conv2d_raw(y, None, H * W * Cin, wd, ops.N.f32(y), H * W * Cout, B, H, W, Cin, Cout, 1,
                           res_ptr=ops.N.f32(res, 'residual'), res_bs=H * W * Cout, w_tc=wtc, x_planes=planes)
            out['y'] = y
    elif route in ('project_dgrad', 'expand_dgrad_fp32', 'lateral_dgrad'):
        operand = x.view(M, Cin).double()

        def launch():
            out['y'] = ops.conv2d(x, wd, Cout, 1, residual=res, w_tc=wtc)
    else:                                       # lateral_fwd: ConvBiasActFn, bias, no activation
        bias = _randn(g, Cout) * 0.1
        operand = x.view(M, Cin).double()
        epi['fn'] = lambda prod: dict(y=prod + bias.double())

        def launch():
            out['y'] = ops.conv2d(x, wf, Cout, 1, bias=bias, act=ops.ACT_NONE, w_tc=wtc)
    if 'fn' not in epi:
        epi['fn'] = lambda prod: dict(y=prod + (res.double().view(M, Cout) if res is not None else 0.0))

    def run():
        with _nan_outputs(ops):
            launch()
        return {k: v.view(M, -1) for k, v in out.items()}
    return dict(call=call, B=B, H=H, W=W, Cin=Cin, Cout=Cout, M=M, operand=operand, weight=weight, epi=epi, run=run,
                launch=launch)


def _trace(fn, out_dir, kernel):
    """run fn under torch.profiler -> [(kernel name, grid, shared memory bytes)] of the launches whose name contains
    `kernel`; a launch without a grid or shared-memory field fails.  After dozens of profiler sessions in one process
    a session now and then records no kernel activity at all, so a trace without the kernel is taken again, up to three
    times (fn must be repeatable); a kernel that is never launched still fails"""
    from torch.profiler import ProfilerActivity, profile
    path = pathlib.Path(out_dir) / ('%s.json' % kernel)
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        prof.export_chrome_trace(str(path))
        with open(path) as f:
            events = json.load(f)['traceEvents']
        out = []
        for e in events:
            if e.get('cat') == 'kernel' and kernel in e.get('name', ''):
                args = e.get('args', {})
                assert 'grid' in args and 'shared memory' in args, ('the trace lacks a field of', e['name'], args)
                out.append((e['name'].replace(' ', ''), list(args['grid']), int(args['shared memory'])))
        if out:
            return out
    raise AssertionError('no %s launch in three traces' % kernel)


def _sra_setup(B, HW, C):
    g = _gen(B * 7 + HW + C)
    a = _randn(g, B, HW, C)
    z = _randn(g, B, HW, C) * 2
    sc, sh = _rand(g, C) + 0.5, _randn(g, C) * 0.3
    out = torch.zeros(B, C, device=_dev())

    def launch():
        from models import _native as N
        N.call('effdet_spatial_reduce_act', a, N.f32(a), N.f32(z), N.f32(sc), N.f32(sh), N.f32(out), 1.0, B, HW, C)
    return dict(a=a, z=z, sc=sc, sh=sh, out=out, launch=launch)


def _record_launches(out_dir):
    """run every pw_gemm and spatial_reduce_act call of the GPU tests once under torch.profiler; write {case: [(name,
    grid, shared memory)]} to out_dir/launches.json"""
    from models import _ops as ops
    ops.PRECISION = 'bf16x3'
    rec = {}
    for B, HW, C in _sra_cases():
        s = _sra_setup(B, HW, C)
        rec['sra %d %d %d' % (B, HW, C)] = _trace(s['launch'], out_dir, 'spatial_reduce_kernel')
        del s
    for case in PW_CASES:
        s = _pw_setup(ops, case)
        rec[str(case)] = _trace(s['launch'], out_dir, 'pw_gemm_kernel')
        del s
    with open(pathlib.Path(out_dir) / 'launches.json', 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def launches(tmp_path_factory):
    """the kernel names, grids and shared memory of every call below, recorded by _record_launches in a fresh
    interpreter: a CUDA activity trace in a long test process can miss this library's kernels"""
    out = tmp_path_factory.mktemp('pw_se_launches')
    here = os.path.dirname(os.path.abspath(__file__))
    repo = os.path.dirname(here)
    path = [here, os.path.join(repo, 'oracle'), os.path.join(repo, 'efficientdet.pytorch_b200'), repo]
    code = 'import sys; sys.path[:0] = %r; import test_pointwise_se_parity as T; T._record_launches(%r)' % (path, str(out))
    subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], check=True, cwd=repo,
                   timeout=1200)
    with open(out / 'launches.json') as f:
        return {k: [(n, tuple(grid), smem) for n, grid, smem in v] for k, v in json.load(f).items()}


# ------------------------------------------------------------------------------------------------
# 1. pw_gemm_kernel at the benchmark's layers
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', PW_CASES, ids=['%s-%s-%s' % c for c in PW_CASES])
def test_pw_gemm_at_benchmark_layers(ops, case, launches):
    """one pw_gemm call with the epilogue fields its route uses, into NaN-filled outputs, against the operand times the
    weight in float64 on the device: whole tensor, each image, each 64-column block.  Controls: the neighbouring
    image's gate on the second image's rows of shared tiles, the last column block without its last k-block, hi*hi only"""
    s = _pw_setup(ops, case)
    B, Cin, Cout, M = s['B'], s['Cin'], s['Cout'], s['M']
    got = s['run']()
    prod = s['operand'] @ s['weight'].t()
    want = s['epi']['fn'](prod)
    plan = _plan_of(s['call'], _sms())
    what = '%s %s %s %d->%d B=%d %dx%d: KB %d, BN %d x %d n-tiles, %s weights, NS %d, %d units per CTA, %d images per tile' \
        % (case[0], case[1], case[2], Cin, Cout, B, s['H'], s['W'], plan['KB'], plan['BN'], plan['ntn'],
           'resident' if plan['bres'] else 'streamed', plan['NS'], plan['upc'], plan['images'])
    print(what)
    errs = {}
    for k, w in want.items():
        assert torch.isfinite(got[k]).all(), (what, k, 'NaN or inf in the output')
        errs[k] = _pw_errs(got[k], w, B)
        print('  %s: rel err %.2e (bound %.0e), worst image %.2e, worst 64-column block %.2e (bound %.0e)'
              % (k, errs[k][0], TOL_TC, errs[k][1], errs[k][2], TOL_ROW))
    # launch plan
    ln = launches[str(case)]
    assert len(ln) == 1, ln
    name, grid, smem = ln[0]
    assert 'pw_gemm_kernel<%d>(' % plan['NB'] in name and grid == plan['grid'] and smem == plan['smem'], (ln, plan)
    for k, (e, img, blk) in errs.items():
        assert e < TOL_TC and img < TOL_ROW and blk < TOL_ROW, (what, k, errs[k])
    # controls, on the raw product output (z of the project forward)
    key = 'z' if 'z' in want else 'y'
    k0, n0 = 64 * (plan['KB'] - 1), (Cout - 1) // 64 * 64
    miss = want[key].clone()
    miss[:, n0:] -= s['operand'][:, k0:] @ s['weight'][n0:, k0:].t()
    ctrl_k = _pw_errs(got[key], miss, B)[2]
    hihi = s['operand'].to(torch.bfloat16).double() @ s['weight'].to(torch.bfloat16).double().t()
    ctrl_hh = _rel(hihi, prod)
    msg = '  controls: last column block without its last k-block %.2e, hi*hi only %.2e' % (ctrl_k, ctrl_hh)
    assert ctrl_k > TOL_ROW and ctrl_hh > TOL_TC, (ctrl_k, ctrl_hh)
    if case[2] == 'project_fwd' and plan['images'] > 1:
        HW = s['H'] * s['W']
        m = torch.arange(M, device=_dev())
        img = m // HW
        first = (m // 128 * 128) // HW
        nb = torch.where(img > first, img - 1, img)
        q, gate = s['epi']['q'], s['epi']['gate']
        op_nb = _swish(q).view(M, Cin) * gate.double()[nb]
        ctrl_gate = max(_rel(a, b) for a, b in zip(got['z'].view(B, -1, Cout),
                                                    (op_nb @ s['weight'].t()).view(B, -1, Cout)))
        msg += ', neighbouring image\'s gate %.2e' % ctrl_gate
        assert ctrl_gate > TOL_ROW, ctrl_gate
    print(msg)


# ------------------------------------------------------------------------------------------------
# 2. the squeeze-excite gate
# ------------------------------------------------------------------------------------------------

def _se_inputs(B, C, S):
    g = _gen(B * 100003 + C * 7 + S)
    mean = _rand(g, B, C) * 1.5 - 0.25             # means of swish activations
    w1, b1 = _randn(g, S, C) / C ** 0.5, _randn(g, S) * 0.1
    w2, b2 = _randn(g, C, S) * (1.5 / S ** 0.5), _randn(g, C) * 0.1
    dgate = _randn(g, B, C)
    return g, mean, w1, b1, w2, b2, dgate


@pytest.mark.gpu
@pytest.mark.parametrize('B,C,S', _se_shapes())
def test_se_gate(B, C, S):
    """effdet_se_gate_fwd / effdet_se_gate_bwd against float64 autograd: s_pre, gate and dmean per image, dW1 and dW2 per
    row, db1, db2; the weight gradients accumulate into non-zero buffers; two backward calls are bit-identical.
    Controls (B > 1): s_pre from the wrong image's mean, dW2 without the last image, dp2 without (1 - g)"""
    from models import _native as N
    g, mean, w1, b1, w2, b2, dgate = _se_inputs(B, C, S)
    s_pre = torch.full((B, S), float('nan'), device=_dev())
    gate = torch.full((B, C), float('nan'), device=_dev())
    N.call('effdet_se_gate_fwd', mean, N.f32(mean), N.f32(w1), N.f32(b1), N.f32(w2), N.f32(b2), N.f32(s_pre),
           N.f32(gate), B, C, S)
    leaves = [t.double().requires_grad_(True) for t in (mean, w1, b1, w2, b2)]
    sp = leaves[0] @ leaves[1].t() + leaves[2]
    gt = torch.sigmoid(_swish(sp) @ leaves[3].t() + leaves[4])
    (gt * dgate.double()).sum().backward()
    dmean_r, dw1_r, db1_r, dw2_r, db2_r = [t.grad for t in leaves]
    sp, gt = sp.detach(), gt.detach()

    def rows(got, want):
        """the worst row's norm-relative error (NaN in got propagates and fails the bound)"""
        return float(((got.double() - want).norm(dim=1) / want.norm(dim=1)).max())

    def bwd():
        # non-zero accumulators, each row of the magnitude of its reference row: the kernel adds into them
        acc = []
        for seed, ref in enumerate((dw1_r, db1_r, dw2_r, db2_r)):
            rms = ref.norm(dim=-1, keepdim=True) / ref.shape[-1] ** 0.5
            acc.append((_randn(_gen(seed), *ref.shape) * rms).float())
        dw = [t.clone() for t in acc]
        dmean = torch.full((B, C), float('nan'), device=_dev())
        ws = torch.full((B * (C + S),), float('nan'), device=_dev())
        N.call('effdet_se_gate_bwd', mean, N.f32(dgate), N.f32(mean), N.f32(s_pre), N.f32(gate), N.f32(w1), N.f32(w2),
               N.f32(dmean), N.f32(dw[0]), N.f32(dw[1]), N.f32(dw[2]), N.f32(dw[3]), N.f32(ws), B, C, S)
        return dmean, [d.double() - a.double() for d, a in zip(dw, acc)], dw, ws
    dmean, (dw1, db1, dw2, db2), raw1, ws1 = bwd()
    dmean2, _, raw2, ws2 = bwd()
    dp2, dp1 = ws1[:B * C].view(B, C), ws1[B * C:].view(B, S)
    dp2_r = dgate.double() * gt * (1 - gt)
    dp1_r = (dp2_r @ w2.double()) * torch.autograd.functional.vjp(_swish, sp, torch.ones_like(sp))[1]
    # a row of dW1 or dW2 is a sum over the batch of dp1[b, j] mean[b, :] or dp2[b, c] swish(s_pre[b, :]): with one or
    # two images its relative error is that of single dp1 / dp2 elements, which a near-cancelling sum over C (dp1) or a
    # gate near 1 (dp2) makes ill-conditioned.  So se_bwd_dw_kernel's rows are held to float64 of its own fp32 inputs
    # (dp1, dp2 from the workspace, mean, s_pre), and dp1, dp2 per image and dW1, dW2 whole to float64 autograd
    dw1_k = dp1.double().t() @ mean.double()
    dw2_k = dp2.double().t() @ _swish(s_pre.double())
    errs = dict(s_pre=rows(s_pre, sp), gate=rows(gate, gt), dp2=rows(dp2, dp2_r), dp1=rows(dp1, dp1_r),
                dmean=rows(dmean, dmean_r), dW1=_rel(dw1, dw1_r), dW2=_rel(dw2, dw2_r), dW1_rows=rows(dw1, dw1_k),
                dW2_rows=rows(dw2, dw2_k), db1=_rel(db1, db1_r), db2=_rel(db2, db2_r))
    print('se (B, C, S) = (%d, %d, %d): %s (bound %.0e)' % (B, C, S, ', '.join('%s %.2e' % kv for kv in errs.items()),
                                                            TOL_EXACT))
    assert max(errs.values()) < TOL_EXACT, errs
    same = torch.equal(dmean, dmean2) and all(torch.equal(a, b) for a, b in zip(raw1, raw2)) and torch.equal(ws1, ws2)
    assert same, 'two backward calls differ'
    if B > 1:
        sp_wrong = mean.double().roll(1, 0) @ w1.double().t() + b1.double()
        c_mean = rows(s_pre, sp_wrong)
        c_dw2 = rows(dw2, dw2_k - dp2[-1].double()[:, None] * _swish(s_pre[-1].double())[None, :])
        c_dp2 = _rel(db2, (gt * dgate.double()).sum(0))
        print('  controls: wrong image\'s mean %.2e, dW2 without the last image %.2e, dp2 without (1 - g) %.2e'
              % (c_mean, c_dw2, c_dp2))
        assert min(c_mean, c_dw2, c_dp2) > TOL_EXACT, (c_mean, c_dw2, c_dp2)


# ------------------------------------------------------------------------------------------------
# 3. spatial_reduce_act
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('B,HW,C', _sra_cases())
def test_spatial_reduce_act(B, HW, C, launches):
    """dgate[b, c] = sum_r dq[b, r, c] * swish(z[b, r, c] * scale[c] + shift[c]) into a zeroed buffer, each image's row
    against float64; the grid against _row_grid; control: one image without its first row block"""
    s = _sra_setup(B, HW, C)
    s['launch']()
    act = _swish(s['z'].double() * s['sc'].double() + s['sh'].double())
    want = (s['a'].double() * act).sum(1)
    grid, rpb = _row_grid(HW, C // 4, B, _sms())
    worst = max(_rel(a, b) for a, b in zip(s['out'], want))
    ctrl_want = want.clone()
    ctrl_want[0] -= (s['a'][0, :rpb].double() * act[0, :rpb]).sum(0)
    ctrl = max(_rel(a, b) for a, b in zip(s['out'], ctrl_want))
    ln = launches['sra %d %d %d' % (B, HW, C)]
    print('spatial_reduce_act (B, HW, C) = (%d, %d, %d): grid %s, %d rows per block: worst image %.2e (bound %.0e); '
          'control without one row block %.2e' % (B, HW, C, grid, rpb, worst, TOL_SUM, ctrl))
    assert len(ln) == 1 and ln[0][1] == grid, (ln, grid)
    assert worst < TOL_SUM, worst
    assert ctrl > TOL_SUM, ctrl


# ------------------------------------------------------------------------------------------------
# 4. MBConvFn composed, against fp64 autograd of O.mbconv_forward
# ------------------------------------------------------------------------------------------------

def _block_state(config, i):
    from bench import CONFIGS
    c = CONFIGS[config]
    cfg = O.make_config(c['net'], num_classes=c['K'], W_bifpn=c['W'], D_bifpn=c['D'])
    q = 'backbone._blocks.%d.' % i
    spec = [(n, shape, kind) for n, shape, kind in O.state_dict_spec(cfg) if n.startswith(q)]
    g = torch.Generator().manual_seed(1000 + i)
    sd = {}
    for n, shape, kind in spec:
        if kind == 'bn_n':
            continue
        if kind == 'conv':
            fan = shape[1] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * (1.5 / fan ** 0.5)
        elif kind == 'bn_w':
            t = torch.rand(shape, generator=g) * 0.6 + 0.7
        elif kind == 'bn_rv':
            t = torch.rand(shape, generator=g) + 0.6
        else:
            t = torch.randn(shape, generator=g) * 0.2
        sd[n] = t.to(_dev())
    return c, cfg, cfg['blocks'][i], q, sd


@pytest.mark.gpu
@pytest.mark.parametrize('config,block,drop', MB_CASES, ids=['%s-%s-%s' % c for c in MB_CASES])
def test_mbconv_block_composed(ops, config, block, drop):
    """MBConvFn forward and backward at the benchmark's B and map against float64 autograd of O.mbconv_forward on the
    device: the output, the input gradient and every parameter gradient, each against its own bound"""
    i = _resolve_block(config, block)
    c, cfg, blk, q, sd = _block_state(config, i)
    B = c['bs']
    H, W = _stem_out(c['size'], c['size'])
    for j in range(i):
        b_ = cfg['blocks'][j]
        H, W = _dw_out(b_['k'], b_['s'], H, W)
    g = _gen(77 + i)
    x = _randn(g, B, H, W, blk['cin'])
    k, s = blk['k'], blk['s']
    left, right, top, bottom = O.same_pad(k, s, cfg['nominal'])          # MBConvBlock._kernel_cfg
    kcfg = dict(k=k, s=s, eps=O.BN_EPS, expand=blk['e'] != 1, skip=blk['skip'], pad_t=top, pad_l=left,
                pad_h=top + bottom, pad_w=left + right)
    rate = O.DROP_CONNECT_RATE * i / len(cfg['blocks'])
    keep = None
    if drop:                    # drop_connect_scale's floor(kp + u) / kp, with image 0 dropped and image 1 kept
        kp = 1 - rate
        keep = torch.floor(kp + _rand(g, B)) / kp
        keep[0], keep[1] = 0.0, 1.0 / kp
    names = ([q + '_expand_conv.weight'] + [q + '_bn0.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
             if kcfg['expand'] else [])
    names += [q + '_depthwise_conv.weight'] + [q + '_bn1.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
    names += [q + '_se_reduce.weight', q + '_se_reduce.bias', q + '_se_expand.weight', q + '_se_expand.bias',
              q + '_project_conv.weight'] + [q + '_bn2.' + n for n in ('weight', 'bias', 'running_mean', 'running_var')]
    params = [sd[n].clone().requires_grad_('running' not in n) for n in names]
    xg = x.clone().requires_grad_(True)
    y = ops.MBConvFn.apply(xg, keep, kcfg, *params)
    dy = _randn(g, *y.shape)
    y.backward(dy)
    # float64 reference: the same parameters, NCHW; drop-connect as the multiplier keep (floor(kp + u) / kp)
    sd64 = {n: v.double().requires_grad_('running' not in n) for n, v in sd.items()}
    x64 = x.permute(0, 3, 1, 2).double().requires_grad_(True)
    y64 = O.mbconv_forward(sd64, q, blk, x64, cfg['nominal'])
    if keep is not None:                  # drop-connect with the same per-image multiplier floor(kp + u) / kp
        y64 = (y64 - x64) * keep.double().view(B, 1, 1, 1) + x64
    y64.backward(dy.permute(0, 3, 1, 2).double())
    errs = {'y': _rel(y.detach().permute(0, 3, 1, 2), y64.detach()), 'dx': _rel(xg.grad.permute(0, 3, 1, 2), x64.grad)}
    for n, p in zip(names, params):
        if p.requires_grad:
            errs[n[len(q):]] = _rel(p.grad, sd64[n].grad)
    print('mbconv %s block %d (B %d, %dx%d, %d->%d, drop-connect %s): %s (bounds %.0e / %.0e)'
          % (config, i, B, H, W, blk['cin'], blk['cout'], drop, ', '.join('%s %.2e' % kv for kv in errs.items()),
             TOL_MB_FWD, TOL_MB_GRAD))
    assert errs['y'] < TOL_MB_FWD, errs
    assert max(v for n, v in errs.items() if n != 'y') < TOL_MB_GRAD, errs
