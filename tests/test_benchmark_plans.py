"""Kernel parity at the launch plans the benchmark reaches.

Several launchers choose their schedule from the problem size: pw_wgrad_launch (pw_wgrad.cu) how many pixel chunks one
CTA accumulates, pick_tiles_per_cta (dw_fused.cu) how many spatial tiles one depthwise CTA loops over, effdet_stem_wgrad
(stem.cu) how many 64-pixel row segments one CTA strides over and which TPG instantiation runs.  The other kernel tests
run at small batches and maps, where these plans are mostly the trivial ones.  This file

  * mirrors the three launchers' arithmetic in Python (_pw_plan, _dw_plan, _stem_plan);
  * walks every MBConv layer and the stem of bench.CONFIGS and checks, without a GPU, that the cases below reach every
    plan the benchmark reaches (test_cases_reach_benchmark_plans);
  * runs each case once under torch.profiler and compares the grid of the launch with the mirror's;
  * holds each kernel to a float64 reference at those plans, with a negative control that shows the bound has teeth.

Bounds (norm-relative error ||got - want|| / ||want||):
  TOL_TC    = 3e-5  bf16x3 weight gradient, whole tensor (as tests/test_planes_path_parity.py)
  TOL_ROW   = 1e-4  the same on every output-channel row of a pointwise weight gradient
  TOL_DW    = 5e-5  the fp32 depthwise kernels (as test_dwconv_fused_forward_backward), whole tensors and each image's
                    squeeze-excite mean row and each tap of the depthwise weight gradient
  TOL_EXACT = 5e-6  fp32 element-wise outputs of the stem and of bnact_bwd
  TOL_SUM   = 2e-5  fp32 sums over many atomic blocks (stem weight gradient, BN affine gradients)

The pointwise weight gradient at the benchmark's layers, measured on an H100 80GB HBM3 (700 W): whole tensor / worst
output-channel row, and the pixels one CTA accumulates.  With one wave of CTAs and no cap, as pw_wgrad_launch had it:
  d0 block 0 project 32->16              16 000 pixels   5.19e-5 / 6.51e-5
  d0 block 1 expand 16->96, dy planes    15 904          5.60e-5 / 8.02e-5
  d4 block 2 expand 24->144, dy planes   15 936          5.53e-5 / 7.21e-5
  d4 block 2 expand 24->144, dy fp32     15 936          5.53e-5 / 7.23e-5
With at most kWgMaxPixelsPerSplit = 4 096 pixels per CTA (tc_ptx.cuh):
  d0 block 0 project                      4 096          1.45e-5 / 1.69e-5
  d0 block 1 expand, dy planes            4 000          1.46e-5 / 2.03e-5
  d4 block 2 expand, dy planes            4 032          1.41e-5 / 1.98e-5
  d4 block 2 expand, dy fp32              4 032          1.41e-5 / 1.99e-5"""
import json

import pytest
import torch
import torch.nn.functional as F

import effdet_oracle as O
from test_planes_path_parity import _box

TOL_TC = 3e-5
TOL_ROW = 1e-4
TOL_DW = 5e-5
TOL_EXACT = 5e-6
TOL_SUM = 2e-5

SMS = 132                       # H100 SXM: the SM count the benchmark's plans are walked at
BN_EPS = 1e-3


def _cdiv(a, b):
    return -(-a // b)


def _dev():
    return torch.device('cuda:0')


def _rel(got, want):
    return float((got - want).norm() / want.norm())


# ------------------------------------------------------------------------------------------------
# mirrors of the launchers
# ------------------------------------------------------------------------------------------------

PW_MAX_PIXELS = 4096            # kWgMaxPixelsPerSplit (tc_ptx.cuh)


def _pw_plan(B, H, W, Cin, Cout, sms, cap=PW_MAX_PIXELS):
    """pw_wgrad_launch (pw_wgrad.cu): tiles, pixels per chunk K, chunks, chunks per split, splits, the kernel's NB and the
    pixels one CTA accumulates.  cap=None: without the cap on pixels per CTA"""
    M = B * H * W
    ntn = _cdiv(Cin, 128)
    NX = _cdiv(_cdiv(Cin, ntn), 16) * 16
    ntn = _cdiv(Cin, NX)
    ntm = _cdiv(Cout, 128)
    TM = _cdiv(_cdiv(Cout, ntm), 8) * 8
    ntm = _cdiv(Cout, TM)
    tiles = ntn * ntm
    octs = min(NX, Cin) // 8 + TM // 8
    K = 128
    while K > 16 and K * octs > 256 * 3:            # kWgCT * kWgUnits converter units per stage
        K >>= 1
    nchunks = _cdiv(M, K)
    splits = max(1, sms // tiles)
    if cap is not None:
        need = _cdiv(nchunks, cap // K)
        if splits < need:
            splits = _cdiv(need * tiles, sms) * sms // tiles
    splits = min(splits, nchunks)
    cps = _cdiv(nchunks, splits)
    splits = _cdiv(nchunks, cps)
    return dict(tiles=tiles, K=K, nchunks=nchunks, cps=cps, splits=splits, NB=2 if NX > 64 else 1, pixels=K * cps,
                grid=(tiles, splits, 1))


DW_TOTAL_PAD = {(3, 1): 2, (3, 2): 1, (5, 1): 4, (5, 2): 3}     # the reference's static padding (nominal sizes are even)


def _dw_out(k, s, H, W):
    t = DW_TOTAL_PAD[(k, s)]
    return (H + t - k) // s + 1, (W + t - k) // s + 1


def _pick_tiles_per_cta(ntiles, other):
    """pick_tiles_per_cta (dw_fused.cu), with its fixed 148 * 6 * 3"""
    return max(1, min((ntiles * other) // (148 * 6 * 3), 8, ntiles))


def _dw_plan(direction, k, s, C, H, W, B):
    """tile grid of effdet_dwconv_fwd_fused / effdet_dwconv_bwd_fused (dw_fused.cu)"""
    Ho, Wo = _dw_out(k, s, H, W)
    if direction == 'fwd':
        ry, rx = Ho, Wo
    else:                                           # backward: tiles of cells (one cell = s x s input pixels)
        ry, rx = _cdiv(H, s), _cdiv(W, s)
    small = ry <= 8 and rx <= 8
    ty = (8 if s == 1 else 4) if small else (16 if s == 1 else 8)
    tx = 8 if small else 16
    tiles_x, tiles_y = _cdiv(rx, tx), _cdiv(ry, ty)
    ntiles = tiles_x * tiles_y
    chunks = _cdiv(C // 4, 4)
    tpc = _pick_tiles_per_cta(ntiles, chunks * B)
    return dict(small=small, tile=(ty, tx), ntiles=ntiles, tpc=tpc, partial=ntiles % tpc != 0,
                grid=(chunks, _cdiv(ntiles, tpc), B))


def _stem_out(H, W):
    return (H - 2) // 2 + 1, (W - 2) // 2 + 1


def _stem_plan(B, H, W, C0, sms):
    """grid and TPG of effdet_stem_wgrad (stem.cu)"""
    Ho, Wo = _stem_out(H, W)
    segs = _cdiv(Wo, 64)
    units = B * Ho * segs
    blocks = min(units, sms * 8)
    tgs = 32 // (C0 // 4)
    tpg = _cdiv(27, tgs)
    return dict(tpg=7 if tpg <= 7 else 9 if tpg <= 9 else 14, grid=(blocks, 1, 1), segs_per_cta=_cdiv(units, blocks),
                partial=Wo % 64 != 0)


# ------------------------------------------------------------------------------------------------
# the benchmark's layers
# ------------------------------------------------------------------------------------------------

def _bench_layers(name):
    """the pointwise weight gradients, depthwise launches and stem of one bench.CONFIGS entry: forward and backward for
    the train configs, forward for the inference one"""
    from bench import CONFIGS
    c = CONFIGS[name]
    cfg = O.make_config(c['net'], num_classes=c['K'], W_bifpn=c['W'], D_bifpn=c['D'])
    B, train = c['bs'], c['mode'] == 'train'
    dirs = ('fwd', 'bwd') if train else ('fwd',)
    pw, dw = [], []
    H, W = _stem_out(c['size'], c['size'])
    stem = dict(C0=cfg['stem'], B=B, H=c['size'], W=c['size'], train=train)
    for i, blk in enumerate(cfg['blocks']):
        mid = blk['cin'] * blk['e']
        pre = blk['e'] != 1
        if pre and train:            # the expand conv's dy arrives as bf16 planes when its map has a pixel box
            mode = 'planes' if mid % 8 == 0 and _box(B, H, W) is not None else 'plain'
            pw.append(dict(block=i, mode=mode, shape=(B, H, W, blk['cin'], mid)))
        for d in dirs:
            dw.append(dict(block=i, dir=d, k=blk['k'], s=blk['s'], pre=pre, shape=(mid, H, W, B)))
        H, W = _dw_out(blk['k'], blk['s'], H, W)
        if train:
            pw.append(dict(block=i, mode='project', shape=(B, H, W, mid, blk['cout'])))
    return pw, dw, stem


# ------------------------------------------------------------------------------------------------
# the GPU cases
# ------------------------------------------------------------------------------------------------

# pointwise weight gradient: (B, H, W, Cin, Cout, mode) -- the benchmark's longest K ranges in each mode.  The benchmark
# has no plain expand (every map has a pixel box), so the plain case is d4 block 2 with dy in fp32: the route the
# expand takes when its map has none
PW_CASES = {
    'd0_block0_project': (32, 256, 256, 32, 16, 'project'),
    'd0_block1_expand_planes': (32, 256, 256, 16, 96, 'planes'),
    'd4_block2_expand_planes': (4, 512, 512, 24, 144, 'planes'),
    'd4_block2_expand_plain': (4, 512, 512, 24, 144, 'plain'),
}

# depthwise: (k, s, BN0, C, H, W, benchmark batch or None).  The first five are bench d0's blocks 0-4; B is the smallest
# batch whose forward and backward plans match the benchmark's (tiles per CTA, partial last group).  The last three are
# the templates the benchmark runs only with BN0, without it at odd sizes; B is the smallest batch with more than one
# tile per CTA in both directions
DW_CASES = {
    'd0_block0': (3, 1, False, 32, 256, 256, 32),
    'd0_block1': (3, 2, True, 96, 256, 256, 32),
    'd0_block2': (3, 1, True, 144, 128, 128, 32),
    'd0_block3': (5, 2, True, 144, 128, 128, 32),
    'd0_block4': (5, 1, True, 240, 64, 64, 32),
    'k3s2_no_bn0': (3, 2, False, 32, 250, 262, None),
    'k5s1_no_bn0': (5, 1, False, 48, 120, 136, None),
    'k5s2_no_bn0': (5, 2, False, 64, 190, 254, None),
}

# stem: (C0, H, W, B).  bench d0 and d4 at their real shapes, the other widths of B0-B7 at odd sizes
STEM_CASES = {
    'b0_d0_bench': (32, 512, 512, 32),
    'b3_odd': (40, 300, 301, 3),
    'b4_d4_bench': (48, 1024, 1024, 4),
    'b6_odd': (56, 385, 515, 2),
    'b7_odd': (64, 200, 131, 5),
}


def _dw_batch(case):
    k, s, _, C, H, W, Bb = DW_CASES[case]

    def key(B):
        return [(p['tpc'], p['partial']) for p in (_dw_plan(d, k, s, C, H, W, B) for d in ('fwd', 'bwd'))]
    for B in range(1, (Bb or 64) + 1):
        if (Bb is not None and key(B) == key(Bb)) or (Bb is None and min(t for t, _ in key(B)) > 1):
            return B
    raise AssertionError('no batch reaches the plan of %s' % case)


def _dw_class(d, k, s, pre, p):
    return (d, k, s, pre, p['small'])


def test_cases_reach_benchmark_plans():
    """every plan class the benchmark reaches is reached by a GPU case below, and the mirrors reproduce the figures that
    motivated them (132 SMs)"""
    pw, dw, stems = [], [], []
    for name in ('d0', 'd4', 'd7'):
        p, d, st = _bench_layers(name)
        pw += p
        dw += d
        stems.append(st)

    # pointwise: the longest K range of each mode, without and with the cap; with it no layer exceeds the cap
    assert _pw_plan(32, 256, 256, 32, 16, SMS, cap=None)['pixels'] == 16000
    assert _pw_plan(32, 256, 256, 16, 96, SMS, cap=None)['pixels'] == 15904
    assert _pw_plan(4, 512, 512, 24, 144, SMS, cap=None)['pixels'] == 15936
    assert _pw_plan(32, 256, 256, 32, 16, SMS)['grid'] == (1, 512, 1)
    modes = {l['mode'] for l in pw}
    assert modes == {'project', 'planes'}, modes
    for cap in (None, PW_MAX_PIXELS):
        for mode in ('project', 'planes', 'plain'):
            bench = [_pw_plan(*l['shape'], SMS, cap=cap)['pixels'] for l in pw if l['mode'] == mode]
            cases = [_pw_plan(*c[:5], SMS, cap=cap)['pixels'] for c in PW_CASES.values() if c[5] == mode]
            assert cases and max(cases) >= max(bench, default=0), (mode, cap, bench, cases)
    assert max(_pw_plan(*l['shape'], SMS)['pixels'] for l in pw) <= PW_MAX_PIXELS
    assert max(_pw_plan(*l['shape'], SMS, cap=None)['pixels'] for l in pw) > 3 * PW_MAX_PIXELS

    # depthwise: the benchmark's block-0 plan, then every (direction, k, s, BN0, SMALL) class with more than one tile per
    # CTA -- and every (k, s) template with and without BN0 -- the cap of 8 and a partial last group
    p0 = _dw_plan('fwd', 3, 1, 32, 256, 256, 32)
    assert (p0['ntiles'], p0['tpc'], p0['ntiles'] % p0['tpc']) == (256, 6, 4)
    bench_plans = [(l, _dw_plan(l['dir'], l['k'], l['s'], *l['shape'])) for l in dw]
    bench_cls = {_dw_class(l['dir'], l['k'], l['s'], l['pre'], p) for l, p in bench_plans if p['tpc'] > 1}
    case_plans = []
    for case, (k, s, pre, C, H, W, _) in DW_CASES.items():
        B = _dw_batch(case)
        for d in ('fwd', 'bwd'):
            case_plans.append(((d, k, s, pre), _dw_plan(d, k, s, C, H, W, B)))
    case_cls = {_dw_class(*c, p) for c, p in case_plans if p['tpc'] > 1}
    templates = {(d, k, s, pre, False) for d in ('fwd', 'bwd') for k, s in DW_TOTAL_PAD for pre in (False, True)}
    assert bench_cls <= case_cls and templates <= case_cls, (bench_cls - case_cls, templates - case_cls)
    assert max(p['tpc'] for _, p in bench_plans) == 8 and max(p['tpc'] for _, p in case_plans) == 8
    assert any(p['partial'] for _, p in bench_plans) and any(p['partial'] and p['tpc'] > 1 for _, p in case_plans)
    for case, c in DW_CASES.items():
        if c[6] is not None:
            assert _dw_batch(case) <= c[6]
    assert _dw_plan('fwd', 3, 1, 32, 256, 256, _dw_batch('d0_block0'))['tpc'] == 6

    # stem: each TPG instantiation and every width of B0-B7, the benchmark's segments per CTA, a partial last segment
    plans = {c: _stem_plan(B, H, W, C0, SMS) for c, (C0, H, W, B) in STEM_CASES.items()}
    assert {p['tpg'] for p in plans.values()} == {7, 9, 14}
    # B0-B6 through the detectors; no detector maps to B7 (width 2.0)
    widths = {O.make_config('efficientdet-d%d' % i)['stem'] for i in range(8)} | {O._round_filters(32, 2.0)}
    assert widths == {32, 40, 48, 56, 64} and widths <= {c[0] for c in STEM_CASES.values()}
    bench_stem = [_stem_plan(st['B'], st['H'], st['W'], st['C0'], SMS) for st in stems if st['train']]
    assert {st['C0'] for st in stems if st['train']} <= {c[0] for c in STEM_CASES.values()}
    assert max(p['segs_per_cta'] for p in plans.values()) >= max(max(p['segs_per_cta'] for p in bench_stem), 8)
    assert any(p['partial'] and STEM_CASES[c][2] % 2 for c, p in plans.items())


# ------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ------------------------------------------------------------------------------------------------

def _launches(fn, tmp_path, kernel):
    """run fn once under torch.profiler; -> [(kernel name, grid)] of the launches whose name contains `kernel`"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = tmp_path / ('%s.json' % kernel)
    prof.export_chrome_trace(str(path))
    with open(path) as f:
        events = json.load(f)['traceEvents']
    out = []
    for e in events:
        if e.get('cat') == 'kernel' and kernel in e.get('name', ''):
            assert 'grid' in e.get('args', {}), ('the trace records no grid for', e['name'])
            out.append((e['name'].replace(' ', ''), tuple(e['args']['grid'])))
    assert out, ('no %s launch in the trace' % kernel)
    return out


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


# ------------------------------------------------------------------------------------------------
# 1. pointwise weight gradient (pw_wgrad_kernel)
# ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize('case', list(PW_CASES))
def test_pointwise_wgrad_at_benchmark_k_ranges(case, tmp_path):
    """dW += dy^T act(x) at the benchmark's layers, accumulated into a non-zero dw, against float64; control: a reference
    without the first 4 096 pixels"""
    from models import _ops as ops
    B, H, W, Cin, Cout, mode = PW_CASES[case]
    g = _gen(Cin * 1000 + Cout + B)
    x = _randn(g, B, H, W, Cin)
    dy = _randn(g, B, H, W, Cout)
    sc, sh = _rand(g, Cin) + 0.5, _randn(g, Cin) * 0.3
    gate = _rand(g, B, Cin)

    def act(b, rows=slice(None)):
        a = x[b].reshape(-1, Cin)[rows].double()
        if mode == 'project':
            a = _swish(a * sc.double() + sh.double()) * gate[b].double()
        return a
    ref = torch.zeros(Cout, Cin, dtype=torch.float64, device=_dev())
    for b in range(B):
        ref += dy[b].reshape(-1, Cout).double().t() @ act(b)
    first = dy[0].reshape(-1, Cout)[:PW_MAX_PIXELS].double().t() @ act(0, slice(0, PW_MAX_PIXELS))
    dw0 = _randn(g, Cout, Cin, 1, 1) * float(ref.std())
    dw = dw0.clone()
    if mode == 'planes':
        assert ops.planes_ok(B, H, W, Cout)
        hi = dy.to(torch.bfloat16)
        planes = torch.stack([hi, (dy - hi.float()).to(torch.bfloat16)]).contiguous()
        del hi

        def launch():
            ops.conv_wgrad_raw(x, ops.N.f32(x), H * W * Cin, None, H * W * Cout, dw, None, B, H, W, Cin, Cout, 1, tc=True,
                               dy_planes=planes)
    elif mode == 'project':
        def launch():
            ops.conv_wgrad(x, dy, dw, None, 1, a_scale=gate, tc=True, in_scale=sc, in_shift=sh)
    else:
        def launch():
            ops.conv_wgrad(x, dy, dw, None, 1, tc=True)
    got_launch = _launches(launch, tmp_path, 'pw_wgrad_kernel')
    got = (dw.double() - dw0.double()).view(Cout, Cin)
    plan = _pw_plan(B, H, W, Cin, Cout, _sms())

    def errs(want):
        rows = ((got - want).norm(dim=1) / want.norm(dim=1)).max()
        return _rel(got, want), float(rows)
    e, row = errs(ref)
    ctrl, ctrl_row = errs(ref - first)
    print('pw wgrad %s %d->%d B=%d %dx%d: %d pixels per CTA (%d splits): rel err %.2e (bound %.0e), worst row %.2e '
          '(bound %.0e); control without %d pixels %.2e / %.2e'
          % (mode, Cin, Cout, B, H, W, plan['pixels'], plan['splits'], e, TOL_TC, row, TOL_ROW, PW_MAX_PIXELS, ctrl,
             ctrl_row))
    assert len(got_launch) == 1 and got_launch[0][1] == plan['grid'], (got_launch, plan)
    assert 'pw_wgrad_kernel<%d>(' % plan['NB'] in got_launch[0][0], got_launch
    assert e < TOL_TC and row < TOL_ROW, (e, row)
    assert ctrl > TOL_TC and ctrl_row > TOL_ROW, (ctrl, ctrl_row)


# ------------------------------------------------------------------------------------------------
# 2. depthwise forward and backward (dw_fwd_fused_kernel, dw_bwd_fused_kernel)
# ------------------------------------------------------------------------------------------------

def _dw_reference(x, wd, bn, gate, dq, dmean, k, s, pre, mask=None):
    """test_dwconv_fused_forward_backward's autograd formula in float64 for ONE image (NHWC device tensors), output
    gradients optionally masked; -> z1, mean, dx, dw, [dgamma1, dbeta1, dgamma0, dbeta0]"""
    t = DW_TOTAL_PAD[(k, s)]
    pt = (k - 1) // 2 if s == 1 else (0 if k == 3 else 1)
    xr = x.permute(2, 0, 1)[None].double().requires_grad_(True)
    wr = wd.double().requires_grad_(True)
    gam = [b_['g'].double().requires_grad_(True) for b_ in bn]
    bet = [b_['b'].double().requires_grad_(True) for b_ in bn]

    def bnf(v, i):
        return F.batch_norm(v, bn[i]['m'].double(), bn[i]['v'].double(), gam[i], bet[i], False, 0.0, BN_EPS)
    a0 = _swish(bnf(xr, 0)) if pre else xr
    z1 = F.conv2d(F.pad(a0, (pt, t - pt, pt, t - pt)), wr, None, s, 0, 1, wd.shape[0])
    a1 = _swish(bnf(z1, 1))
    HW = z1.shape[2] * z1.shape[3]
    gout = gate.double()[None, :, None, None] * dq.permute(2, 0, 1)[None].double() + dmean.double()[None, :, None, None] / HW
    if mask is not None:
        gout = gout * mask
    (a1 * gout).sum().backward()
    bn_grads = [gam[1].grad, bet[1].grad] + ([gam[0].grad, bet[0].grad] if pre else [])
    return (z1.detach()[0].permute(1, 2, 0), a1.detach().mean(dim=(0, 2, 3)), xr.grad[0].permute(1, 2, 0), wr.grad,
            bn_grads)


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(DW_CASES))
def test_dwconv_fused_multi_tile_plans(case, tmp_path):
    """z1 and the squeeze-excite mean (each image's row), then dx, dW (each tap) and both BN affines, at plans with
    several tiles per CTA, against float64 autograd on the device image by image; controls: one image's mean without
    one forward tile, dW without the output gradient of one backward tile"""
    from models import _native as N
    k, s, pre, C, H, W, _ = DW_CASES[case]
    B = _dw_batch(case)
    pt = (k - 1) // 2 if s == 1 else (0 if k == 3 else 1)
    Ho, Wo = _dw_out(k, s, H, W)
    g = _gen(k * 100 + s * 10 + C + H)
    x = _randn(g, B, H, W, C)
    wd = _randn(g, C, 1, k, k) / k
    bn = [dict(g=_rand(g, C) + 0.5, b=_randn(g, C) * 0.3, m=_randn(g, C) * 0.3, v=_rand(g, C) + 0.5) for _ in range(2)]
    gate = _rand(g, B, C)
    dq = _randn(g, B, Ho, Wo, C)
    dmean = _randn(g, B, C)

    def fold(i):
        rstd = 1.0 / torch.sqrt(bn[i]['v'] + BN_EPS)
        sc = bn[i]['g'] * rstd
        return [t.contiguous() for t in (sc, bn[i]['b'] - bn[i]['m'] * sc, bn[i]['m'], rstd)]
    sc0, sh0, mu0, rs0 = fold(0)
    sc1, sh1, mu1, rs1 = fold(1)
    wkkc = wd.view(C, k * k).t().contiguous()
    z1 = torch.full((B, Ho, Wo, C), float('nan'), device=_dev())
    mean = torch.zeros(B, C, device=_dev())
    fa = N.DwFwdArgs(N.f32(x), N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(wkkc), N.f32(sc1),
                     N.f32(sh1), N.f32(z1), N.f32(mean), B, H, W, C, k, s, pt, pt, Ho, Wo, 1.0 / (Ho * Wo))
    dx = torch.full((B, H, W, C), float('nan'), device=_dev())
    dw = torch.zeros(C, 1, k, k, device=_dev())
    dgb = torch.zeros(4, C, device=_dev())
    ba = N.DwBwdArgs(N.f32(dq), N.f32(z1), N.f32(gate), N.f32(dmean), N.f32(sc1), N.f32(sh1), N.f32(mu1), N.f32(rs1),
                     N.f32(x), N.f32(sc0) if pre else None, N.f32(sh0) if pre else None, N.f32(mu0) if pre else None,
                     N.f32(rs0) if pre else None, N.f32(wkkc), N.f32(dx), N.f32(dw), N.f32(dgb[0]), N.f32(dgb[1]),
                     N.f32(dgb[2]) if pre else None, N.f32(dgb[3]) if pre else None, 1.0 / (Ho * Wo), B, H, W, C, k, s,
                     pt, pt, Ho, Wo, None)
    fwd_launch = _launches(lambda: N.call('effdet_dwconv_fwd_fused', x, fa), tmp_path, 'dw_fwd_fused_kernel')
    bwd_launch = _launches(lambda: N.call('effdet_dwconv_bwd_fused', x, ba), tmp_path, 'dw_bwd_fused_kernel')

    # float64 reference, image by image; the sums over images in float64
    sq = dict(z1=0.0, z1_ref=0.0, dx=0.0, dx_ref=0.0)
    mean_ref = torch.zeros(B, C, dtype=torch.float64, device=_dev())
    dw_ref = torch.zeros(C, 1, k, k, dtype=torch.float64, device=_dev())
    bn_ref = None
    for b in range(B):
        z_r, m_r, dx_r, dw_r, bg_r = _dw_reference(x[b], wd, bn, gate[b], dq[b], dmean[b], k, s, pre)
        sq['z1'] += float((z1[b].double() - z_r).norm()) ** 2
        sq['z1_ref'] += float(z_r.norm()) ** 2
        sq['dx'] += float((dx[b].double() - dx_r).norm()) ** 2
        sq['dx_ref'] += float(dx_r.norm()) ** 2
        mean_ref[b] = m_r
        dw_ref += dw_r
        bn_ref = bg_r if bn_ref is None else [a + c for a, c in zip(bn_ref, bg_r)]
    fp = _dw_plan('fwd', k, s, C, H, W, B)
    bp = _dw_plan('bwd', k, s, C, H, W, B)
    errs = dict(z1=(sq['z1'] / sq['z1_ref']) ** 0.5, dx=(sq['dx'] / sq['dx_ref']) ** 0.5,
                mean_rows=max(_rel(mean[b].double(), mean_ref[b]) for b in range(B)),
                dw=_rel(dw.double(), dw_ref),
                dw_taps=max(_rel(dw.double().view(C, -1)[:, t], dw_ref.view(C, -1)[:, t]) for t in range(k * k)))
    for i, n in enumerate(['dgamma1', 'dbeta1', 'dgamma0', 'dbeta0'][:len(bn_ref)]):
        errs[n] = _rel(dgb[i].double(), bn_ref[i])
    # controls: image 0's mean without the first forward tile; dW without the output gradient of the first backward tile
    ty, tx = fp['tile']
    z_r, _, _, _, _ = _dw_reference(x[0], wd, bn, gate[0], dq[0], dmean[0], k, s, pre)
    a1 = _swish(z_r * sc1.double() + sh1.double())
    ctrl_mean = _rel(mean[0].double(), mean_ref[0] - a1[:ty, :tx].sum(dim=(0, 1)) / (Ho * Wo))
    mask = torch.ones(Ho, Wo, dtype=torch.float64, device=_dev())
    cy, cx = bp['tile']
    mask[:cy, :cx] = 0
    dw_full0 = _dw_reference(x[0], wd, bn, gate[0], dq[0], dmean[0], k, s, pre)[3]
    dw_drop0 = _dw_reference(x[0], wd, bn, gate[0], dq[0], dmean[0], k, s, pre, mask=mask)[3]
    want_ctrl = (dw_ref - dw_full0 + dw_drop0).view(C, -1)
    ctrl_tap = max(_rel(dw.double().view(C, -1)[:, t], want_ctrl[:, t]) for t in range(k * k))
    print('dw %s k%d s%d BN0=%s C=%d %dx%d B=%d: fwd %d tiles per CTA (of %d), bwd %d (of %d); %s (bound %.0e); '
          'controls: mean without a tile %.2e, dW without a tile %.2e'
          % (case, k, s, pre, C, H, W, B, fp['tpc'], fp['ntiles'], bp['tpc'], bp['ntiles'],
             ', '.join('%s %.2e' % kv for kv in errs.items()), TOL_DW, ctrl_mean, ctrl_tap))
    tmpl = '%d,%d,%s,%s>' % (k, s, str(pre).lower(), '%s')
    assert len(fwd_launch) == 1 and fwd_launch[0][1] == fp['grid'], (fwd_launch, fp)
    assert 'dw_fwd_fused_kernel<' + tmpl % str(fp['small']).lower() in fwd_launch[0][0], fwd_launch
    assert len(bwd_launch) == 1 and bwd_launch[0][1] == bp['grid'], (bwd_launch, bp)
    assert 'dw_bwd_fused_kernel<' + tmpl % str(bp['small']).lower() in bwd_launch[0][0], bwd_launch
    assert max(errs.values()) < TOL_DW, errs
    assert ctrl_mean > TOL_DW and ctrl_tap > TOL_DW, (ctrl_mean, ctrl_tap)


# ------------------------------------------------------------------------------------------------
# 3. stem and its BatchNorm (stem_fwd_px_kernel, bnact_bwd_kernel, stem_wgrad_kernel)
# ------------------------------------------------------------------------------------------------

def _bn_params(g, C):
    gamma, beta = _rand(g, C) + 0.5, _randn(g, C) * 0.3
    mu, var = _randn(g, C) * 0.3, _rand(g, C) + 0.5
    rstd = 1.0 / torch.sqrt(var + BN_EPS)
    scale = gamma * rstd
    return gamma, beta, mu, var, scale.contiguous(), (beta - mu * scale).contiguous(), rstd.contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(STEM_CASES))
def test_stem_forward_bn_backward_wgrad(case, tmp_path):
    """effdet_stem_fwd (z and y), effdet_bnact_bwd in SWISH mode, effdet_stem_wgrad, against F.pad(x, (0,1,0,1)), a
    stride-2 conv and BN + swish in float64 on the device; control: dW without the last 64-pixel row segment"""
    from models import _native as N, _ops as ops
    C0, H, W, B = STEM_CASES[case]
    Ho, Wo = _stem_out(H, W)
    g = _gen(C0 * 7 + H + W + B)
    x = _randn(g, B, 3, H, W)
    w = _randn(g, C0, 3, 3, 3) * (1.5 / 27 ** 0.5)
    gamma, beta, mu, var, scale, shift, rstd = _bn_params(g, C0)
    dy = _randn(g, B, Ho, Wo, C0)
    z = torch.full((B, Ho, Wo, C0), float('nan'), device=_dev())
    y = torch.full((B, Ho, Wo, C0), float('nan'), device=_dev())
    N.call('effdet_stem_fwd', x, N.f32(x), N.f32(w), N.f32(scale), N.f32(shift), N.f32(z), N.f32(y), B, H, W, C0)
    dz, dgamma, dbeta = ops.bnact_bwd(dy, z, scale, shift, mu, rstd, ops.ACT_SWISH)
    dw = torch.zeros(C0, 3, 3, 3, device=_dev())
    launch = _launches(lambda: N.call('effdet_stem_wgrad', x, N.f32(x), N.f32(dz), N.f32(dw), B, H, W, C0), tmp_path,
                       'stem_wgrad_kernel')

    sq = {n: [0.0, 0.0] for n in ('z', 'y', 'dz')}
    dw_ref = torch.zeros(C0, 3, 3, 3, dtype=torch.float64, device=_dev())
    dg_ref = torch.zeros(C0, dtype=torch.float64, device=_dev())
    db_ref = torch.zeros_like(dg_ref)
    G = 4
    for b0 in range(0, B, G):
        sl = slice(b0, min(B, b0 + G))
        xp = F.pad(x[sl].double(), (0, 1, 0, 1))
        wr = w.double().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        zr = F.conv2d(xp, wr, None, 2)
        zr.retain_grad()
        u = (zr - mu.double()[:, None, None]) / torch.sqrt(var.double()[:, None, None] + BN_EPS) * gr[:, None, None] + \
            br[:, None, None]
        yr = _swish(u)
        (yr * dy[sl].permute(0, 3, 1, 2).double()).sum().backward()
        for n, got, want in (('z', z[sl], zr), ('y', y[sl], yr), ('dz', dz[sl], zr.grad)):
            want = want.detach().permute(0, 2, 3, 1)
            sq[n][0] += float((got.double() - want).norm()) ** 2
            sq[n][1] += float(want.norm()) ** 2
        dw_ref += wr.grad
        dg_ref += gr.grad
        db_ref += br.grad
        if b0 + G >= B:                 # control: the last row segment of the last image (a partial one when Wo % 64)
            seg = torch.zeros_like(zr.grad[-1:])
            ox0 = (Wo - 1) // 64 * 64
            seg[..., -1, ox0:] = zr.grad[-1:, :, -1, ox0:]
            last_seg = torch.nn.grad.conv2d_weight(xp[-1:], w.shape, seg, 2)
    plan = _stem_plan(B, H, W, C0, _sms())
    errs = {n: (a / b) ** 0.5 for n, (a, b) in sq.items()}
    sums = dict(dw=_rel(dw.double(), dw_ref), dgamma=_rel(dgamma.double(), dg_ref), dbeta=_rel(dbeta.double(), db_ref))
    ctrl = _rel(dw.double(), dw_ref - last_seg)
    print('stem %s C0=%d %dx%d B=%d: TPG %d, %d segments per CTA; %s (bound %.0e); %s (bound %.0e); control without '
          'the last segment %.2e' % (case, C0, H, W, B, plan['tpg'], plan['segs_per_cta'],
                                     ', '.join('%s %.2e' % kv for kv in errs.items()), TOL_EXACT,
                                     ', '.join('%s %.2e' % kv for kv in sums.items()), TOL_SUM, ctrl))
    assert len(launch) == 1 and launch[0][1] == plan['grid'], (launch, plan)
    assert 'stem_wgrad_kernel<%d>(' % plan['tpg'] in launch[0][0], launch
    assert max(errs.values()) < TOL_EXACT, errs
    assert max(sums.values()) < TOL_SUM, sums
    assert ctrl > TOL_SUM, ctrl


@pytest.mark.gpu
def test_bnact_bwd_project_bn_row_scale():
    """effdet_bnact_bwd in NONE mode with a per-image row_scale (every project conv's BN2 with drop-connect), at bench
    d0's block-0 project output; control: the affine gradients without image 0's first row"""
    from models import _ops as ops
    B, H, W, C = 32, 256, 256, 16
    g = _gen(2024)
    dy, z = _randn(g, B, H, W, C), _randn(g, B, H, W, C) * 2
    _, _, mu, _, scale, shift, rstd = _bn_params(g, C)
    row = _rand(g, B) + 0.5
    row[3] = 0.0                    # a dropped image
    dz, dgamma, dbeta = ops.bnact_bwd(dy, z, scale, shift, mu, rstd, ops.ACT_NONE, row_scale=row)
    gr = dy.double() * row.double()[:, None, None, None]
    xh = (z.double() - mu.double()) * rstd.double()
    errs = dict(dz=_rel(dz.double(), gr * scale.double()))
    dg_ref, db_ref = (gr * xh).sum(dim=(0, 1, 2)), gr.sum(dim=(0, 1, 2))
    errs.update(dgamma=_rel(dgamma.double(), dg_ref), dbeta=_rel(dbeta.double(), db_ref))
    ctrl = min(_rel(dgamma.double(), dg_ref - (gr[0, 0] * xh[0, 0]).sum(dim=0)), _rel(dbeta.double(), db_ref - gr[0, 0].sum(dim=0)))
    print('bnact_bwd NONE + row_scale %s: %s; control without one row %.2e' % ((B, H, W, C), errs, ctrl))
    assert errs['dz'] < TOL_EXACT and errs['dgamma'] < TOL_SUM and errs['dbeta'] < TOL_SUM, errs
    assert ctrl > TOL_SUM, ctrl
