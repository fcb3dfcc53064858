"""The reference's training loop (train.py:95-133) replayed as one CUDA graph per micro-step: GraphedTrainStep with
FusedClipAdamW bound to it.  The optimizer's learning rate and step count live in device memory, gradients accumulate
over --grad_accumulation_steps micro-steps, and a micro-step whose loss is exactly zero is skipped on the device.

Every bound below has a negative control: a deliberately defective reference (today's frozen bias correction, an
update on a zero loss, an ignored learning-rate change) whose distance from the product must exceed the bound."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
TOL_OPT = 5e-6          # the fused optimizer against fp32 / fp64 AdamW (test_fused_clip_adamw_matches_torch's bound)
SHAPES = [(1,), (7,), (33, 31), (256, 64, 3, 3), (65537,), (300001,), (16,)]


def _dev():
    return torch.device('cuda:0')


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float(torch.linalg.vector_norm(a - b) / max(float(torch.linalg.vector_norm(b)), 1e-30))


# ------------------------------------------------------------------------------------------------------------------
# CPU: argument refusals of the new entry points
# ------------------------------------------------------------------------------------------------------------------

def test_new_entry_points_refuse_bad_arguments():
    from models import _native
    _native.build()
    lib = _native.load()

    def err():
        return lib.effdet_last_error().decode()

    fake = 1 << 20                                           # aligned non-null "pointer"; never dereferenced
    assert lib.effdet_multi_accumulate(None, fake, fake, fake, fake, 1, 64, fake, None, None, 0, None) == -1
    assert 'multi_accumulate' in err()
    assert lib.effdet_multi_accumulate(fake, fake, fake, fake, fake, 1, 64, None, None, None, 0, None) == -1
    assert 'multi_accumulate' in err()
    assert lib.effdet_multi_accumulate(fake, fake, fake, fake, fake, 0, 64, fake, None, None, 0, None) == -1
    assert 'multi_accumulate' in err()
    assert lib.effdet_multi_accumulate(fake, fake, fake, fake, fake, 1, 64, fake, None, fake, 0, None) == -1
    assert 'multi_accumulate' in err() and 'update_requested' in err()
    good = [fake] * 7 + [1, 64, fake, 0.1, fake, fake, fake, fake, 0.9, 0.999, 1e-8, 1e-2]
    for i in (0, 1, 2, 3, 4, 5, 6, 9, 11, 12, 13, 14):        # every pointer
        args = list(good)
        args[i] = None
        assert lib.effdet_multi_clip_adamw_dev(*args, 0, None) == -1 and 'multi_clip_adamw_dev' in err(), i
    for i, bad in ((7, 0), (8, 0), (15, 1.0), (16, -0.5)):     # nchunks, chunk, beta1, beta2
        args = list(good)
        args[i] = bad
        assert lib.effdet_multi_clip_adamw_dev(*args, 0, None) == -1 and 'multi_clip_adamw_dev' in err(), i
    assert 'betas' in err()


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level: the entry points against fp64 AdamW on the CPU
# ------------------------------------------------------------------------------------------------------------------

class _Kernels:
    """The two new launches plus the existing norm over the chunk tables FusedClipAdamW builds."""

    def __init__(self, ps, lr, step0):
        from models.fused_optim import _chunk_table
        self.ps = ps
        self.accs = [torch.zeros_like(p) for p in ps]
        self.gs = [torch.zeros_like(p) for p in ps]
        self.ms = [torch.zeros_like(p) for p in ps]
        self.vs = [torch.zeros_like(p) for p in ps]
        self.tab = _chunk_table(ps, p=ps, acc=self.accs, g=self.gs, m=self.ms, v=self.vs)
        self.lr = torch.tensor([lr], dtype=torch.float32, device=_dev())
        self.step = torch.tensor([step0], dtype=torch.int64, device=_dev())
        self.update = torch.ones((1,), dtype=torch.int32, device=_dev())
        self.gate = torch.zeros((1,), dtype=torch.int32, device=_dev())
        self.ticket = torch.zeros((1,), dtype=torch.int32, device=_dev())
        self.norm_sq = torch.zeros((1,), dtype=torch.float32, device=_dev())
        self.loss = torch.ones((1,), dtype=torch.float32, device=_dev())

    def accumulate(self, loss, update=True):
        from models import _native as N
        self.loss.fill_(loss)
        self.update.fill_(1 if update else 0)
        t = self.tab
        N.call('effdet_multi_accumulate', self.lr, t['acc'].data_ptr(), t['g'].data_ptr(), t['numels'].data_ptr(),
               t['ct'].data_ptr(), t['co'].data_ptr(), t['nchunks'], 65536, self.loss.data_ptr(),
               self.update.data_ptr(), self.gate.data_ptr())

    def update_step(self, max_norm, betas=(0.9, 0.999), eps=1e-8, wd=1e-2):
        from models import _native as N
        t = self.tab
        self.norm_sq.zero_()
        N.call('effdet_multi_sumsq', self.lr, t['acc'].data_ptr(), t['numels'].data_ptr(), t['ct'].data_ptr(),
               t['co'].data_ptr(), t['nchunks'], 65536, self.norm_sq.data_ptr())
        N.call('effdet_multi_clip_adamw_dev', self.lr, t['p'].data_ptr(), t['acc'].data_ptr(), t['m'].data_ptr(),
               t['v'].data_ptr(), t['numels'].data_ptr(), t['ct'].data_ptr(), t['co'].data_ptr(), t['nchunks'], 65536,
               self.norm_sq.data_ptr(), max_norm, self.lr.data_ptr(), self.step.data_ptr(), self.gate.data_ptr(),
               self.ticket.data_ptr(), betas[0], betas[1], eps, wd)

    def snapshot(self):
        return [t.clone() for t in self.ps + self.ms + self.vs + self.accs + [self.step]]


def _adamw_fp64(p, m, v, grads, lr, t, max_norm, b1=0.9, b2=0.999, eps=1e-8, wd=1e-2):
    """clip_grad_norm_ + torch.optim.AdamW in fp64; t = the 1-based step the bias corrections use"""
    norm = float(np.sqrt(sum(float((g.double() ** 2).sum()) for g in grads)))
    coef = min(1.0, max_norm / (norm + 1e-6))
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    for i, g in enumerate(grads):
        g = g.double() * coef
        p[i] = p[i] * (1.0 - lr * wd)
        m[i] = b1 * m[i] + (1.0 - b1) * g
        v[i] = b2 * v[i] + (1.0 - b2) * g * g
        p[i] = p[i] - lr / bc1 * m[i] / (v[i].sqrt() / np.sqrt(bc2) + eps)


@pytest.mark.gpu
@pytest.mark.parametrize('step0', [0, 1000])
def test_gated_update_matches_fp64_adamw(step0):
    """12 gated steps with a learning rate that changes every step, the counter starting at 0 and at a loaded value.
    Two micro-batches accumulate per step; a closed gate in between changes nothing."""
    g = torch.Generator().manual_seed(7)
    p0 = [torch.randn(s, generator=g) for s in SHAPES]
    k = _Kernels([p.clone().to(_dev()) for p in p0], lr=1e-2, step0=step0)
    ref_p = [p.double() for p in p0]
    ref_m = [torch.zeros_like(p) for p in ref_p]
    ref_v = [torch.zeros_like(p) for p in ref_p]
    frozen = ([p.clone() for p in ref_p], [m.clone() for m in ref_m], [v.clone() for v in ref_v])   # control
    max_norm = 0.1
    for it in range(12):
        lr = 1e-2 * 0.8 ** it
        k.lr.fill_(lr)
        grads = []
        for micro in range(2):
            gm = [torch.randn(s, generator=g) * (0.5 + it) for s in SHAPES]
            for src, dst in zip(gm, k.gs):
                dst.copy_(src)
            k.accumulate(loss=1.0, update=micro == 1)
            grads = gm if micro == 0 else [a + b for a, b in zip(grads, gm)]
            if micro == 0:                                    # gate closed: the launch must change nothing
                before = k.snapshot()
                k.update_step(max_norm)
                for a, b in zip(before, k.snapshot()):
                    assert torch.equal(a, b)
        for acc, s in zip(k.accs, grads):                   # the fp32 sum of both micro-batches
            assert torch.equal(acc.cpu(), s)
        k.update_step(max_norm)
        torch.cuda.synchronize()
        acc_sum = [a.double() for a in grads]
        _adamw_fp64(ref_p, ref_m, ref_v, acc_sum, lr, step0 + it + 1, max_norm)
        _adamw_fp64(*frozen, acc_sum, lr, step0 + 4, max_norm)          # today's graph: bias correction of step 4
        assert int(k.step) == step0 + it + 1
        assert all(int(torch.count_nonzero(a)) == 0 for a in k.accs)    # optimizer.zero_grad() after the step
    worst = max(max(_rel(a, b) for a, b in zip(k.ps, ref_p)), max(_rel(a, b) for a, b in zip(k.ms, ref_m)),
                max(_rel(a, b) for a, b in zip(k.vs, ref_v)))
    control = max(_rel(a, b) for a, b in zip(k.ps, frozen[0]))
    print('step0 %d: worst p/m/v rel err %.2e, frozen-bias-correction control %.2e' % (step0, worst, control))
    assert worst < TOL_OPT
    assert control > TOL_OPT


@pytest.mark.gpu
def test_accumulate_is_bit_exact_and_skips_zero_loss():
    g = torch.Generator().manual_seed(8)
    k = _Kernels([torch.randn(s, generator=g).to(_dev()) for s in SHAPES], lr=1e-3, step0=0)
    for acc in k.accs:
        acc.copy_(torch.randn(acc.shape, generator=g))
    for src in k.gs:
        src.copy_(torch.randn(src.shape, generator=g))
    expect = [torch.add(a, b) for a, b in zip(k.accs, k.gs)]
    k.accumulate(loss=0.37, update=True)
    assert all(torch.equal(a, e) for a, e in zip(k.accs, expect))
    assert int(k.gate) == 1
    k.accumulate(loss=0.37, update=False)
    assert int(k.gate) == 0
    before = [a.clone() for a in k.accs]
    for loss in (0.0, -0.0):                                   # bool(loss == 0) holds for both zeros
        k.accumulate(loss=loss, update=True)
        assert all(torch.equal(a, b) for a, b in zip(k.accs, before))
        assert int(k.gate) == 0
    k.accumulate(loss=float('nan'), update=True)               # not zero: the reference backpropagates it too
    assert int(k.gate) == 1


# ------------------------------------------------------------------------------------------------------------------
# GPU, loop level: a small deterministic model with EfficientDet's call interface, graphed vs the literal train.py loop
# ------------------------------------------------------------------------------------------------------------------

class _Tiny(torch.nn.Module):
    """model([images, annotations]) -> (cls_loss[1], reg_loss[1]); both exactly 0 when every annotation row is -1"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(11)
        self.l1 = torch.nn.Linear(48, 32)
        self.l2 = torch.nn.Linear(32, 8)
        self.unused = torch.nn.Parameter(torch.randn(5, generator=g))      # never receives a gradient
        with torch.no_grad():
            for p in (self.l1.weight, self.l1.bias, self.l2.weight, self.l2.bias):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)

    def forward(self, inputs):
        images, annots = inputs
        out = self.l2(torch.tanh(self.l1(images.flatten(1))))
        valid = annots[..., 4] >= 0
        tgt = (annots[..., :4] * valid[..., None]).sum(1)
        w = valid.any(1).float()
        cls = (w * ((out[:, :4] - tgt) ** 2).mean(1)).sum(0, keepdim=True) / images.shape[0]
        reg = (w * (out[:, 4:] - 0.5 * tgt).abs().mean(1)).sum(0, keepdim=True) / images.shape[0]
        return cls, reg


def _tiny_batches(n, zero_at, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        images = torch.randn(4, 3, 4, 4, generator=g)
        ann = torch.rand(4, 3, 5, generator=g)
        ann[1, 2] = -1                                          # padding rows, as the reference's collater writes
        if i in zero_at:
            ann[:] = -1                                         # a batch without annotations: loss exactly 0
        out.append((images.to(_dev()), ann.to(_dev())))
    return out


class _DefectiveAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW's single-tensor arithmetic with one defect: bias corrections frozen at `frozen_step`, or the
    learning rate frozen at its initial value"""

    def __init__(self, params, lr, frozen_step=None, frozen_lr=False):
        super().__init__(params, dict(lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2))
        self.frozen_step, self.lr0 = frozen_step, (lr if frozen_lr else None)

    @torch.no_grad()
    def step(self):
        for group in self.param_groups:
            lr = self.lr0 if self.lr0 is not None else group['lr']
            b1, b2 = group['betas']
            for p in group['params']:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st.update(step=0, exp_avg=torch.zeros_like(p), exp_avg_sq=torch.zeros_like(p))
                st['step'] += 1
                t = self.frozen_step or st['step']
                p.mul_(1 - lr * group['weight_decay'])
                st['exp_avg'].lerp_(p.grad, 1 - b1)
                st['exp_avg_sq'].mul_(b2).addcmul_(p.grad, p.grad, value=1 - b2)
                denom = (st['exp_avg_sq'].sqrt() / (1 - b2 ** t) ** 0.5).add_(group['eps'])
                p.addcdiv_(st['exp_avg'], denom, value=-lr / (1 - b1 ** t))


def _reference_loop(model, opt, batches, k, epochs, skip_zero=True):
    """train.py:95-133, line for line (ReduceLROnPlateau with patience 0; threshold 0.99 so that epoch 2 reduces)"""
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, patience=0, threshold=0.99)
    params, lrs = [], []
    for epoch in range(epochs):
        opt.zero_grad()
        total_loss = []
        for idx, (images, annotations) in enumerate(batches):
            cl, rl = model([images, annotations])
            loss = cl.mean() + rl.mean()
            if skip_zero and bool(loss == 0):
                continue
            loss.backward()
            if (idx + 1) % k == 0:
                torch.nn.utils.clip_grad_norm_(model.parameters(), 0.1)
                opt.step()
                opt.zero_grad()
            total_loss.append(loss.item())
        sched.step(np.mean(total_loss))
        params.append([p.detach().clone() for p in model.parameters()])
        lrs.append(opt.param_groups[0]['lr'])
    return params, lrs


def _graphed_loop(model, opt, batches, k, epochs):
    from models.graph_step import GraphedTrainStep
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, patience=0, threshold=0.99)
    step = GraphedTrainStep(model, batches[0][0], batches[0][1], optimizer=opt)
    params, lrs, losses = [], [], []
    for epoch in range(epochs):
        opt.zero_grad()
        ep = [step(images, annotations, update=(idx + 1) % k == 0).clone() for idx, (images, annotations)
              in enumerate(batches)]
        ep = torch.stack(ep)
        losses.append(ep.cpu())
        sched.step(float(ep[ep != 0].mean()))
        params.append([p.detach().clone() for p in model.parameters()])
        lrs.append(opt.param_groups[0]['lr'])
    return params, lrs, losses


def _worst(a_params, b_params):
    return max(_rel(a, b) for a, b in zip(a_params, b_params) if float(b.abs().max()) > 0)


@pytest.mark.gpu
@pytest.mark.parametrize('k', [1, 3])
def test_graphed_loop_matches_reference_train_loop(k):
    """3 epochs x 7 micro-batches; batch 2 (an accumulation boundary for k=3) and batch 4 (off it) have no
    annotations.  Parameters after every epoch, step counts and moments against torch.optim.AdamW in the reference
    loop; controls: updating on a zero loss, bias correction frozen at step 4, an ignored learning-rate change."""
    from models.fused_optim import FusedClipAdamW
    epochs, lr = 3, 3e-2
    batches = _tiny_batches(7, zero_at=(2, 4), seed=21 + k)
    base = _Tiny().to(_dev())

    ref = copy.deepcopy(base)
    ref_opt = torch.optim.AdamW(ref.parameters(), lr=lr)
    ref_params, ref_lrs = _reference_loop(ref, ref_opt, batches, k, epochs)
    assert ref_lrs[1] < lr and ref_lrs[0] == lr                # the scheduler reduced the lr after epoch 2

    prod = copy.deepcopy(base)
    opt = FusedClipAdamW(prod.parameters(), lr=lr, max_norm=0.1)
    prod_params, prod_lrs, losses = _graphed_loop(prod, opt, batches, k, epochs)
    assert prod_lrs == ref_lrs
    assert all(float(l[2]) == 0.0 and float(l[4]) == 0.0 and float(l[0]) != 0.0 for l in losses)
    for e in range(epochs):
        worst = _worst(prod_params[e], ref_params[e])
        assert worst < TOL_OPT, (e, worst)
    assert torch.equal(prod.unused.detach(), base.unused.detach()) and torch.equal(ref.unused.detach(), base.unused.detach())

    sd, ref_sd = opt.state_dict(), ref_opt.state_dict()
    assert sd['state'].keys() == ref_sd['state'].keys()
    for i, st in sd['state'].items():
        assert int(st['step']) == int(ref_sd['state'][i]['step']), i
        assert _rel(st['exp_avg'], ref_sd['state'][i]['exp_avg']) < TOL_OPT
        assert _rel(st['exp_avg_sq'], ref_sd['state'][i]['exp_avg_sq']) < TOL_OPT
    assert int(next(iter(sd['state'].values()))['step']) == {1: 15, 3: 3}[k]     # boundaries on a zero-loss batch are skipped

    controls = {}
    for name, make, skip in (('updates on zero loss', lambda ps: torch.optim.AdamW(ps, lr=lr), False),
                             ('bias correction frozen at step 4', lambda ps: _DefectiveAdamW(ps, lr, frozen_step=4), True),
                             ('ignores the lr change', lambda ps: _DefectiveAdamW(ps, lr, frozen_lr=True), True)):
        m = copy.deepcopy(base)
        params, _ = _reference_loop(m, make(m.parameters()), batches, k, epochs, skip_zero=skip)
        controls[name] = _worst(prod_params[-1], params[-1])
    print('k=%d: worst per-epoch parameter rel err %.2e, controls %s' % (k, _worst(prod_params[-1], ref_params[-1]),
                                                                       {n: '%.2e' % v for n, v in controls.items()}))
    assert all(v > TOL_OPT for v in controls.values()), controls


@pytest.mark.gpu
def test_building_the_graphed_step_changes_nothing_and_frozen_settings_are_refused():
    from models import _native as N
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    batches = _tiny_batches(2, zero_at=(), seed=31)
    model = _Tiny().to(_dev())
    opt = FusedClipAdamW(model.parameters(), lr=1e-2, max_norm=0.1)
    cl, rl = model(list(batches[0]))
    (cl.mean() + rl.mean()).backward()
    opt.step()                                                  # pre-existing state: step 1, non-zero moments
    del cl, rl
    before = ([p.detach().clone() for p in model.parameters()],
              {id(p): {k: (v.clone() if torch.is_tensor(v) else v) for k, v in st.items()} for p, st in opt.state.items()})
    step = GraphedTrainStep(model, batches[0][0], batches[0][1], optimizer=opt)
    torch.cuda.synchronize()
    for a, b in zip(model.parameters(), before[0]):
        assert torch.equal(a.detach(), b)
    for p, st in opt.state.items():
        for key, v in before[1][id(p)].items():
            assert torch.equal(st[key], v) if torch.is_tensor(v) else st[key] == v, key
    assert {int(st['step']) for st in opt.state_dict()['state'].values()} == {1}
    step(*batches[1])
    assert {int(st['step']) for st in opt.state_dict()['state'].values()} == {2}   # the true count after one replay
    for p, a in zip(model.parameters(), before[0]):
        if p.grad is not None:
            assert int(torch.count_nonzero(p.grad)) == 0          # the accumulators were emptied by the update

    with pytest.raises(N.EffdetNativeError, match='load the optimizer state before'):
        opt.load_state_dict(opt.state_dict())
    with pytest.raises(N.EffdetNativeError, match='bound to a GraphedTrainStep'):
        opt.step()
    group = opt.param_groups[0]
    for key, changed in (('betas', (0.8, 0.999)), ('eps', 1e-6), ('weight_decay', 0.0), ('max_norm', 1.0)):
        keep = group[key]
        group[key] = changed
        with pytest.raises(N.EffdetNativeError, match='fixed in the CUDA graph'):
            step(*batches[1])
        group[key] = keep
    step(*batches[1], update=False)                             # accumulation is allowed with FusedClipAdamW

    plain = GraphedTrainStep(_Tiny().to(_dev()), batches[0][0], batches[0][1])
    with pytest.raises(N.EffdetNativeError, match='needs optimizer=FusedClipAdamW'):
        plain(*batches[1], update=False)
    other = _Tiny().to(_dev())
    other_step = GraphedTrainStep(other, batches[0][0], batches[0][1], optimizer=torch.optim.SGD(other.parameters(), lr=0.1))
    with pytest.raises(N.EffdetNativeError, match='needs optimizer=FusedClipAdamW'):
        other_step(*batches[1], update=False)
    other_step(*batches[1])


# ------------------------------------------------------------------------------------------------------------------
# GPU, whole model: D0 through the eager drop-in loop and through the graphed step
# ------------------------------------------------------------------------------------------------------------------

def _d0(sd):
    from models import EfficientDet
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(sd)
    m = m.to(_dev())
    m.eval()                                                    # drop-connect off: both sides see the same function
    m.is_training = True
    return m


def _d0_eager_loop(m, opt, batches, k, frozen_bias=False):
    losses = []
    opt.zero_grad()
    for idx, (images, annotations) in enumerate(batches):
        cl, rl = m([images, annotations])
        loss = cl.mean() + rl.mean()
        if bool(loss == 0):
            losses.append(0.0)
            continue
        loss.backward()
        if (idx + 1) % k == 0:
            if frozen_bias:                                     # today's graph: every step corrected as step 4
                for st in opt.state.values():
                    st['step'] = 3
            opt.step()
            opt.zero_grad()
        losses.append(loss.item())
    return losses


# measured on an H100 SXM 80 GB HBM3 (700 W limit): update rel err median 1.9e-3, worst 2.7e-1 over 274 updated
# tensors (Adam's normalisation turns gradient noise on near-zero gradients into whole updates); loss rel err 2.9e-5;
# the frozen-bias-correction control at median 1.1e-1
D0_MEDIAN, D0_WORST = 5e-3, 6e-1


@pytest.mark.gpu
def test_graphed_d0_training_matches_eager_drop_in():
    """6 micro-batches, k=2, batch 3 without annotations: the total parameter update of the graphed loop against the
    eager drop-in loop with FusedClipAdamW.  The gradients of the two differ by the order of fp32 atomics, amplified by
    the network's gradient conditioning (DESIGN.md section 2); Adam's normalisation carries that into the updates."""
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=41)
    batches = []
    for s in range(6):
        images, ann = O.synthetic_batch(2, size=256, num_classes=20, seed=50 + s)
        if s == 3:
            ann[:] = -1
        batches.append((images.to(_dev()), ann.to(_dev())))
    k = 2

    def eager(frozen_bias):
        m = _d0(sd)
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        losses = _d0_eager_loop(m, opt, batches, k, frozen_bias)
        torch.cuda.synchronize()
        return {n: p.detach() - p0[n] for n, p in m.named_parameters()}, losses

    upd_e, loss_e = eager(False)
    upd_f, _ = eager(True)
    m = _d0(sd)
    p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    step = GraphedTrainStep(m, batches[0][0], batches[0][1], optimizer=opt)
    opt.zero_grad()
    loss_g = [float(step(images, ann, update=(idx + 1) % k == 0)) for idx, (images, ann) in enumerate(batches)]
    upd_g = {n: p.detach() - p0[n] for n, p in m.named_parameters()}
    assert loss_g[3] == 0.0 and loss_e[3] == 0.0
    errs = sorted(_rel(upd_g[n], upd_e[n]) for n in upd_e if float(upd_e[n].abs().max()) > 0)
    ctrl = sorted(_rel(upd_f[n], upd_e[n]) for n in upd_e if float(upd_e[n].abs().max()) > 0)
    loss_err = max(abs(a - b) / max(abs(b), 1e-30) for a, b in zip(loss_g, loss_e) if b != 0)
    print('D0 graphed vs eager: %d updated tensors, update rel err median %.2e worst %.2e; loss rel err %.2e; '
          'frozen-bias control median %.2e' % (len(errs), errs[len(errs) // 2], errs[-1], loss_err, ctrl[len(ctrl) // 2]))
    assert len(errs) > 250
    assert errs[len(errs) // 2] < D0_MEDIAN and errs[-1] < D0_WORST
    assert loss_err < 1e-3
    assert ctrl[len(ctrl) // 2] > D0_MEDIAN
    assert {int(st['step']) for st in opt.state_dict()['state'].values()} == {2}   # boundaries 1, 3 (no annotations), 5


# ------------------------------------------------------------------------------------------------------------------
# GPU, 2 ranks: DDP + FusedClipAdamW, update=True every call
# ------------------------------------------------------------------------------------------------------------------

def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _ddp_worker(rank, world, port, out):
    os.environ['TORCH_NCCL_ASYNC_ERROR_HANDLING'] = '0'         # torch's recipe for capturing NCCL work
    os.environ['NCCL_ASYNC_ERROR_HANDLING'] = '0'
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    for p in (os.path.join(os.path.dirname(HERE), 'oracle'), os.path.join(os.path.dirname(HERE), 'efficientdet.pytorch_b200')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    from models import _native as N
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=3)
    batches = [O.synthetic_batch(2 * world, size=256, num_classes=20, seed=s_) for s_ in (92, 93, 94)]
    lo, hi = rank * 2, (rank + 1) * 2
    res = {}
    for mode in ('graph', 'eager'):
        from models import EfficientDet
        m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
        m.load_state_dict(sd)
        m = m.to(dev)
        m.eval()
        m.is_training = True
        p0 = {n: p.detach().clone() for n, p in m.named_parameters()}
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            net = torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], find_unused_parameters=True,
                                                            static_graph=True, gradient_as_bucket_view=True,
                                                            broadcast_buffers=False)
        torch.cuda.current_stream(dev).wait_stream(side)
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        if mode == 'graph':
            step = GraphedTrainStep(net, batches[0][0][lo:hi].to(dev), batches[0][1][lo:hi].to(dev), optimizer=opt)
            try:
                step(batches[0][0][lo:hi].to(dev), batches[0][1][lo:hi].to(dev), update=False)
                res['refused'] = False
            except N.EffdetNativeError:
                res['refused'] = True
            for images, ann in batches:
                step(images[lo:hi].to(dev), ann[lo:hi].to(dev))
        else:
            with torch.cuda.stream(side):
                for images, ann in batches:
                    opt.zero_grad()
                    cl, rl = net([images[lo:hi].to(dev), ann[lo:hi].to(dev)])
                    (cl.mean() + rl.mean()).backward()
                    opt.step()
        torch.cuda.synchronize()
        res[mode] = {n: (p.detach() - p0[n]).cpu() for n, p in m.named_parameters()}
        res[mode + '_step'] = int(next(iter(opt.state_dict()['state'].values()))['step'])
    torch.save(res, os.path.join(out, 'r%d.pt' % rank))
    torch.cuda.synchronize()
    dist.barrier(device_ids=[rank])
    os._exit(0)                                                 # (NCCL teardown after a captured collective hangs)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_graphed_update_matches_eager_ddp(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_ddp_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp_path, 'r%d.pt' % r)) for r in (0, 1))
    assert r0['refused'] and r0['graph_step'] == r0['eager_step'] == 3
    errs = []
    for n, ref in r0['eager'].items():
        assert torch.equal(r0['graph'][n], r1['graph'][n]), 'ranks disagree on ' + n
        if float(ref.abs().max()) > 0:
            errs.append(_rel(r0['graph'][n], ref))
    errs.sort()
    print('DDP graphed vs eager: update rel err median %.2e worst %.2e' % (errs[len(errs) // 2], errs[-1]))
    assert errs[len(errs) // 2] < D0_MEDIAN and errs[-1] < D0_WORST
