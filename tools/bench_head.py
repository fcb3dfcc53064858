"""Micro-benchmark of the RetinaHead convolutions as models/_ops.py::RetinaHeadPlanesFn runs them: activations and
gradients as bf16 hi/lo planes, every layer one launch over the five pyramid levels, through the C ABI.  Three shapes:
a 256->256 tower layer, the 256->720 class conv (9 anchors x 80 classes) and a 64->64 BiFPN node conv (D0 width, the
64-column tile of conv_planes_kernel), each in three directions:
  fwd    conv_planes_multi, bias + activation (tower, BiFPN node: ReLU into planes and their mask bits; class conv:
         sigmoid into fp32)
  dgrad  conv_planes_multi on the gradient planes, ReLU mask bits of the layer input, column sums (bias gradient) ->
         planes; dgrad-planes (tower layer only): the same with the mask read from the input's planes
  wgrad  wgrad_planes_multi from the input and gradient planes
and two launches with the same 9-stage mainloop and 256-column output, which differ only in their epilogues: the
forward of a 64->256 first tower layer (D0's BiFPN width) and the data gradient of the 256->36 box conv.
Times are CUDA events around `iters` back-to-back launches; TFLOP/s are algorithmic (2 * pixels * 9 * Cin * Cout per
launch; the tensor cores execute three bf16 products for each).  Every result is also reduced to checksums so that two
builds can be compared.  mode (default bf16x3) selects the precision: bf16 runs the single-pass instances (one bf16
product per multiply-add, the lo planes are not read).
usage: python tools/bench_head.py [B] [size] [iters] [bf16x3|bf16]"""
import os
import subprocess
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200')]
import torch                      # noqa: E402
from models import _native as N   # noqa: E402
from models import _ops as ops    # noqa: E402

B, size, iters = [int(v) for v in (sys.argv[1:4] + ['32', '512', '20'][len(sys.argv) - 1:])[:3]]
mode = sys.argv[4] if len(sys.argv) > 4 else 'bf16x3'
assert mode in ('bf16x3', 'bf16'), mode
ops.PRECISION = mode
dev = torch.device('cuda:0')
g = torch.Generator(device=dev).manual_seed(0)
sides = [size >> s for s in (3, 4, 5, 6, 7)]                  # P3..P7
geo = [(B, s, s) for s in sides]
px = B * sum(s * s for s in sides)
NBUF = 3                                                       # rotating operand sets: every launch misses L2


def planes_of(C, relu=False):
    """random NHWC fp32 maps of every level -> bf16 hi/lo planes (ReLU'd: a tower activation, the dgrad mask)"""
    out = []
    for (b, h, w) in geo:
        x = torch.randn(b, h, w, C, device=dev, generator=g)
        if relu:
            x = x.clamp_min_(0.0)
        p = ops._planes(b, h, w, C, x)
        ops.to_planes(N.f32(x), h * w * C, p, b, h * w, C, x)
        out.append(p)
    return out


def relu_bits(ps, C):
    """the ReLU mask of planes as a forward's y_mask holds it: bit c % 32 of word c // 32 <=> hi + lo > 0"""
    out = []
    for p in ps:
        pos = ((p[0].double() + p[1].double()) > 0)[..., :C]
        nw = (C + 31) // 32
        pos = torch.nn.functional.pad(pos, (0, nw * 32 - C)).reshape(*pos.shape[:-1], nw, 32).long()
        words = (pos << torch.arange(32, device=pos.device)).sum(-1)
        out.append(torch.where(words >= 2 ** 31, words - 2 ** 32, words).int().contiguous())
    return out


def planes_sum(ps):
    return [float(sum((p[0].double() + p[1].double()).sum() for p in ps)),
            float(sum((p[0].double() + p[1].double()).abs().sum() for p in ps))]


def shape(Cin, Cout, act):
    w = torch.randn(Cout, Cin, 3, 3, device=dev, generator=g) / (Cin * 9) ** 0.5
    bias = torch.randn(Cout, device=dev, generator=g)
    tf, td = ops.pack_conv_tc(w)
    xs = [planes_of(Cin, relu=True) for _ in range(NBUF)]     # layer inputs (post-ReLU tower activations)
    dys = [planes_of(Cout) for _ in range(NBUF)]              # gradients w.r.t. the layer outputs
    xbits = [relu_bits(x, Cin) for x in xs]
    if act == N.ACT_RELU:
        ys = [ops._planes(b, h, wd, Cout, w) for (b, h, wd) in geo]
        ybits = [ops._relu_bits(b, h, wd, Cout, w) for (b, h, wd) in geo]
        fwd_lv = [dict(y_planes=ys[l], y_mask=ybits[l]) for l in range(len(geo))]
    else:
        ys = [torch.empty(b, h, wd, Cout, device=dev) for (b, h, wd) in geo]
        fwd_lv = [dict(y_ptr=N.f32(ys[l]), y_bs=geo[l][1] * geo[l][2] * Cout) for l in range(len(geo))]
    dxs = [ops._planes(b, h, wd, Cin, w) for (b, h, wd) in geo]
    colsum = torch.zeros(Cin, device=dev)
    dw = torch.zeros_like(w)

    def fwd(i):
        ops.conv_planes_multi(w, [dict(x=xs[i % NBUF][l], B=b, H=h, W=wd, **fwd_lv[l]) for l, (b, h, wd) in enumerate(geo)],
                              tf, Cin, Cout, 3, bias=bias, act=act)

    def dgrad(i):
        ops.conv_planes_multi(w, [dict(x=dys[i % NBUF][l], y_planes=dxs[l], mask_bits=xbits[i % NBUF][l], B=b, H=h, W=wd)
                                  for l, (b, h, wd) in enumerate(geo)], td, Cout, Cin, 3, colsum=colsum)

    def dgrad_planes(i):
        ops.conv_planes_multi(w, [dict(x=dys[i % NBUF][l], y_planes=dxs[l], mask=xs[i % NBUF][l], B=b, H=h, W=wd)
                                  for l, (b, h, wd) in enumerate(geo)], td, Cout, Cin, 3, colsum=colsum)

    def wgrad(i):
        ops.wgrad_planes_multi(w, [dict(x=xs[i % NBUF][l], dy=dys[i % NBUF][l], B=b, H=h, W=wd)
                                   for l, (b, h, wd) in enumerate(geo)], dw, Cin, Cout, 3)

    def checksum(name):
        colsum.zero_()
        dw.zero_()
        fns[name](0)
        if name == 'fwd':
            if act == N.ACT_RELU:
                assert all(torch.equal(b, r) for b, r in zip(ybits, relu_bits(ys, Cout))), 'y_mask != the planes\' ReLU'
                return planes_sum(ys)
            return [float(sum(y.double().sum() for y in ys)), float(sum(y.double().abs().sum() for y in ys))]
        if name in ('dgrad', 'dgrad-planes'):
            return planes_sum(dxs) + [float(colsum.double().sum())]
        return [float(dw.double().sum()), float(dw.double().abs().sum())]

    fns = {'fwd': fwd, 'dgrad': dgrad, 'dgrad-planes': dgrad_planes, 'wgrad': wgrad}
    return fns, checksum


def timed(fn):
    for i in range(NBUF):
        fn(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


card = subprocess.run(['nvidia-smi', '-i', str(dev.index or 0), '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                      capture_output=True, text=True).stdout.strip()
print('levels', sides, 'B', B, 'pixels', px, 'iters', iters, 'mode', mode, 'card', card)
for Cin, Cout, act, names in ((256, 256, N.ACT_RELU, ('fwd', 'dgrad', 'dgrad-planes', 'wgrad')),
                              (256, 720, N.ACT_SIGMOID, ('fwd', 'dgrad', 'wgrad')), (64, 64, N.ACT_RELU, ('fwd', 'dgrad', 'wgrad')),
                              (64, 256, N.ACT_RELU, ('fwd',)), (256, 36, N.ACT_NONE, ('dgrad',))):
    fns, checksum = shape(Cin, Cout, act)
    flops = 2.0 * px * 9 * Cin * Cout
    for name in names:
        chk = checksum(name)
        ms = timed(fns[name])
        print('%d->%d %-12s %8.3f ms  %6.1f TFLOP/s algorithmic   checksum %s'
              % (Cin, Cout, name, ms, flops / ms / 1e9, ['%.9e' % c for c in chk]), flush=True)
    del fns, checksum
    torch.cuda.empty_cache()
