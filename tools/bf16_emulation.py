"""CPU emulation of EFFDET_B200_PRECISION=bf16 on the fp32 oracle, and what the mode costs in accuracy.

The tensor-core kernels in bf16 mode compute every dense 3x3 convolution of neck and head (groups 1, Cin % 4 == 0,
Cin >= 16: not the stem, not the depthwise convs) from bf16-rounded operands with fp32 accumulation:
    forward  y  = conv(RN(x), RN(w)) + b
    dgrad    dx = convT(RN(dy), RN(w))
    wgrad    dw = corr(RN(x), RN(dy)),   db = sum(dy)  (unrounded)
`BF16Functional` is a stand-in for torch.nn.functional that does exactly that, so swapping it in for the oracle's
module-level `F` turns the fp32 oracle into the reference of the bf16 mode:

    with emulated(O):
        cls, reg = O.train_forward(...)

Run as a script it measures the emulation against the plain oracle (the accuracy cost of the mode):
    python tools/bf16_emulation.py [--quick]
D0 512x512 B=2 train mode (fixed drop-connect samples): neck outputs, cls, reg, both losses, parameter gradients;
D7 1536x1536 inference: neck outputs, cls, reg.  --quick runs D0 at 256x256 only.
"""
import argparse
import contextlib
import os
import sys
import time

import torch
import torch.nn.functional as TF


def rn(t):
    """round to the nearest bf16 value, back in fp32 (the hi plane of the split)"""
    return t.to(torch.bfloat16).to(torch.float32)


class _RoundGrad(torch.autograd.Function):
    """identity whose backward rounds the incoming gradient to bf16 (the dy operand of dgrad and wgrad)"""

    @staticmethod
    def forward(ctx, y):
        return y.view_as(y)

    @staticmethod
    def backward(ctx, g):
        return rn(g)


def single_pass_conv(w, groups=1):
    """does the product run this conv with one bf16 product per multiply-add in bf16 mode?"""
    return groups == 1 and w.dim() == 4 and tuple(w.shape[2:]) == (3, 3) and w.shape[1] % 4 == 0 and w.shape[1] >= 16


class BF16Functional:
    """torch.nn.functional with the dense 3x3 convs replaced by the bf16-mode emulation; round=False switches the
    emulation off (every call is forwarded unchanged)"""

    def __init__(self, round=True):
        self.round = round

    def __getattr__(self, name):
        return getattr(TF, name)

    def conv2d(self, x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
        if not (self.round and single_pass_conv(w, groups)):
            return TF.conv2d(x, w, bias, stride, padding, dilation, groups)
        y = _RoundGrad.apply(TF.conv2d(rn(x), rn(w), None, stride, padding, dilation, groups))
        return y + bias.view(1, -1, 1, 1) if bias is not None else y     # the bias gradient stays unrounded


@contextlib.contextmanager
def emulated(oracle_module, round=True):
    """swap the oracle's module-level F for BF16Functional for the duration of the block"""
    old = oracle_module.F
    oracle_module.F = BF16Functional(round)
    try:
        yield
    finally:
        oracle_module.F = old


def _grad_sd(sd):
    return {k: (v.clone().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v) for k, v in sd.items()}


def d0_train(O, size, B=2):
    """(collect, losses, grads) of one D0 train-mode step with fixed drop-connect samples, plain and emulated"""
    cfg = O.make_config('efficientdet-d0', num_classes=80, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=0)
    images, ann = O.synthetic_batch(B, size=size, num_classes=80, seed=1000)
    g = torch.Generator().manual_seed(4321)
    nskip = sum(1 for i, b in enumerate(cfg['blocks']) if b['skip'] and i > 0)
    keeps = [torch.rand([B, 1, 1, 1], generator=g) for _ in range(nskip)]
    out = []
    for emu in (False, True):
        sdg = _grad_sd(sd)
        col = {}
        ctx = emulated(O) if emu else contextlib.nullcontext()
        with ctx:
            cl, rl = O.train_forward(sdg, images, ann, cfg, keep_samples=keeps, collect=col)
            (cl.mean() + rl.mean()).backward()
        grads = {k: v.grad for k, v in sdg.items() if isinstance(v, torch.Tensor) and v.requires_grad and v.grad is not None}
        out.append((col, (float(cl.detach()), float(rl.detach())), grads))
    return out


def d7_infer(O, size=1536):
    cfg = O.make_config('efficientdet-d7', num_classes=20, W_bifpn=384, D_bifpn=8)
    sd = O.init_state_dict(cfg, seed=51)
    images, _ = O.synthetic_batch(1, size=size, seed=52)
    out = []
    for emu in (False, True):
        col = {}
        ctx = emulated(O) if emu else contextlib.nullcontext()
        with ctx, torch.no_grad():
            O.raw_outputs(sd, images, cfg, collect=col)
        out.append(col)
    return out


def _outputs(O, a, b):
    r = {'neck P%d' % (3 + i): O.rel_err(b['neck'][i], a['neck'][i]) for i in range(len(a['neck']))}
    r['cls'] = O.rel_err(b['cls'], a['cls'])
    r['reg'] = O.rel_err(b['reg'], a['reg'])
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--quick', action='store_true', help='D0 at 256x256 only')
    args = ap.parse_args()
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(repo, 'oracle'))
    import effdet_oracle as O
    torch.set_num_threads(os.cpu_count() or 1)
    size = 256 if args.quick else 512
    t0 = time.time()
    (ca, la, ga), (cb, lb, gb) = d0_train(O, size)
    print('D0 %dx%d B=2 train mode, bf16 emulation vs fp32 oracle (norm-relative):' % (size, size))
    for k, v in _outputs(O, ca, cb).items():
        print('  %-8s %.3e' % (k, v))
    print('  losses   cls %.6f vs %.6f (rel %.3e), reg %.6f vs %.6f (rel %.3e)' % (
        lb[0], la[0], abs(lb[0] - la[0]) / abs(la[0]), lb[1], la[1], abs(lb[1] - la[1]) / abs(la[1])))
    errs = sorted((O.rel_err(gb[k], g), k) for k, g in ga.items() if float(g.abs().max()) > 0)
    print('  param grads: %d, median %.3e, worst %.3e (%s)' % (len(errs), errs[len(errs) // 2][0], errs[-1][0], errs[-1][1]))
    print('  (%.0f s)' % (time.time() - t0))
    if args.quick:
        return
    t0 = time.time()
    a, b = d7_infer(O)
    print('D7 1536x1536 B=1 inference, bf16 emulation vs fp32 oracle (norm-relative):')
    for k, v in _outputs(O, a, b).items():
        print('  %-8s %.3e' % (k, v))
    print('  (%.0f s)' % (time.time() - t0))


if __name__ == '__main__':
    main()
