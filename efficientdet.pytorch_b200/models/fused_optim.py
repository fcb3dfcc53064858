"""Fused ``clip_grad_norm_`` + ``AdamW`` step (SURVEY.md 8(f) rank 1): what the reference's loop does right after
``loss.backward()`` (``train.py:115-118`` with ``optim.AdamW(model.parameters(), lr)``, ``train.py:268``) as two
multi-tensor kernel launches and no host synchronisation.

    opt = FusedClipAdamW(model.parameters(), lr=1e-4, max_norm=0.1)
    loss.backward(); opt.step(); opt.zero_grad()

Semantics follow ``torch.nn.utils.clip_grad_norm_`` (coefficient max_norm / (total_norm + 1e-6), clamped to 1, gradients
rescaled in place) and ``torch.optim.AdamW`` (decoupled weight decay, bias-corrected moments, no amsgrad).

``GraphedTrainStep(..., optimizer=opt)`` binds the optimizer to its CUDA graph.  From then on the optimizer keeps one
step counter and one learning rate per param group in device memory, and ``p.grad`` of every parameter that receives
a gradient is a persistent accumulator that the graph adds each micro-step's gradients to and the update empties.
A bound optimizer: ``state_dict()`` reads the counters back (one device read) and reports the true step count;
``zero_grad()`` zeroes the accumulators in place; ``step()`` and ``load_state_dict()`` are refused (load the state
before building the graphed step).  betas, eps, weight_decay and max_norm are fixed at binding; the learning rate is
re-read from ``param_groups`` before every replay.
"""
import numpy as np
import torch

from . import _native as N

_CHUNK = 65536


def _check_param(p):
    if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or not p.grad.is_contiguous():
        raise N.EffdetNativeError('FusedClipAdamW needs contiguous CUDA float32 parameters and gradients')


def _chunk_table(plist, **tensors):
    """Device tables of one param group: a pointer table per named list of tensors (aligned with plist), the element
    counts, and per chunk of _CHUNK elements the tensor it belongs to and its offset (one CTA per chunk)."""
    dev = plist[0].device
    numels = np.array([p.numel() for p in plist], dtype=np.int64)
    ct, co = [], []
    for t, n in enumerate(numels):
        for off in range(0, int(n), _CHUNK):
            ct.append(t)
            co.append(off)

    def up(a):
        return torch.from_numpy(a).to(dev)

    tab = {k: up(np.array([t.data_ptr() for t in ts], dtype=np.uint64).view(np.int64)) for k, ts in tensors.items()}
    tab.update(numels=up(numels), ct=up(np.array(ct, dtype=np.int32)), co=up(np.array(co, dtype=np.int64)),
               nchunks=len(ct))
    return tab


class FusedClipAdamW(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_norm=0.1):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, max_norm=max_norm)
        super().__init__(params, defaults)
        self._tables = {}
        self.last_norm_sq = None          # device scalar of the most recent step (read it only if you need it)
        self._graph = None                # device-resident state once bound to a CUDA graph (_bind_graph)

    def _table(self, gi, plist):
        ms, vs = [], []
        for p in plist:
            st = self.state[p]
            if 'exp_avg' not in st:
                st['step'] = 0
                st['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            ms.append(st['exp_avg'])
            vs.append(st['exp_avg_sq'])
        # gradients are re-allocated by zero_grad(set_to_none=True) and the moments by load_state_dict():
        # the device tables are rebuilt whenever any of the four pointers of any tensor moved
        key = tuple((p.data_ptr(), p.grad.data_ptr(), m.data_ptr(), v.data_ptr()) for p, m, v in zip(plist, ms, vs))
        hit = self._tables.get(gi)
        if hit is not None and hit[0] == key:
            return hit[1]
        tab = _chunk_table(plist, p=plist, g=[p.grad for p in plist], m=ms, v=vs)
        self._tables[gi] = (key, tab)
        return tab

    @torch.no_grad()
    def step(self, closure=None):
        if self._graph is not None:
            raise N.EffdetNativeError('FusedClipAdamW is bound to a GraphedTrainStep, whose replays run the update; '
                                      'an eager step() would bypass its device-resident step counters')
        loss = closure() if closure is not None else None
        # one global norm over every parameter group, like clip_grad_norm_(model.parameters(), max_norm)
        live = []
        for gi, group in enumerate(self.param_groups):
            plist = [p for p in group['params'] if p.grad is not None]
            for p in plist:
                _check_param(p)
            if plist:
                live.append((gi, group, plist))
        if not live:
            return loss
        dev_t = live[0][2][0]
        norm_sq = torch.zeros((1,), device=dev_t.device, dtype=torch.float32)
        tabs = []
        for gi, group, plist in live:
            tab = self._table(gi, plist)
            tabs.append(tab)
            N.call('effdet_multi_sumsq', dev_t, tab['g'].data_ptr(), tab['numels'].data_ptr(), tab['ct'].data_ptr(),
                   tab['co'].data_ptr(), tab['nchunks'], _CHUNK, norm_sq.data_ptr())
        for (gi, group, plist), tab in zip(live, tabs):
            st0 = self.state[plist[0]]
            # one bias correction per launch: every live parameter of the group must be at the same step (parameters
            # that start receiving gradients later, or checkpoints with per-parameter counts, would silently get the
            # wrong correction -- torch.optim.AdamW tracks the count per parameter)
            steps = {int(self.state[p]['step']) for p in plist}
            if len(steps) > 1:
                raise N.EffdetNativeError('FusedClipAdamW: parameters of one group are at different steps %s; put late '
                                          'starters into their own param group' % sorted(steps))
            step = int(st0['step']) + 1          # int() also accepts the tensor step of a torch.optim.AdamW checkpoint
            for p in plist:
                self.state[p]['step'] = step
            b1, b2 = group['betas']
            N.call('effdet_multi_clip_adamw', dev_t, tab['p'].data_ptr(), tab['g'].data_ptr(), tab['m'].data_ptr(),
                   tab['v'].data_ptr(), tab['numels'].data_ptr(), tab['ct'].data_ptr(), tab['co'].data_ptr(),
                   tab['nchunks'], _CHUNK, norm_sq.data_ptr(), float(group['max_norm'] or 0.0), float(group['lr']),
                   float(b1), float(b2), float(group['eps']), float(group['weight_decay']), 1.0 - b1 ** step,
                   1.0 - b2 ** step, 1)
            # the kernel wrote through raw pointers: tell autograd (and the packed-weight / folded-BN caches of
            # models/_ops.py, which key on Tensor._version) that parameters and gradients changed in place
            torch.autograd.graph.increment_version(plist)
            torch.autograd.graph.increment_version([p.grad for p in plist])
        self.last_norm_sq = norm_sq
        return loss

    # ---- CUDA-graph binding (models/graph_step.py::GraphedTrainStep) ----------------------------------------------

    def _frozen(self):
        return [(tuple(float(b) for b in g['betas']), float(g['eps']), float(g['weight_decay']),
                 float(g['max_norm'] or 0.0)) for g in self.param_groups]

    def _bind_graph(self, live):
        """Before capture: device state for the parameters in `live` (those that receive gradients).  Creates missing
        moments as step() would, and changes no existing value."""
        if self._graph is not None:
            raise N.EffdetNativeError('FusedClipAdamW is already bound to a GraphedTrainStep')
        live_ids = {id(p) for p in live}
        groups, steps = [], []
        for gi, group in enumerate(self.param_groups):
            plist = [p for p in group['params'] if id(p) in live_ids]
            if not plist:
                steps.append(0)
                continue
            for p in plist:
                if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
                    raise N.EffdetNativeError('FusedClipAdamW needs contiguous CUDA float32 parameters')
                st = self.state[p]
                if 'exp_avg' not in st:
                    st['step'] = 0
                    st['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            group_steps = {int(self.state[p]['step']) for p in plist}
            if len(group_steps) > 1:
                raise N.EffdetNativeError('FusedClipAdamW: parameters of one group are at different steps %s; put late '
                                          'starters into their own param group' % sorted(group_steps))
            steps.append(group_steps.pop())
            accs = [torch.zeros_like(p, memory_format=torch.contiguous_format) for p in plist]
            tab = _chunk_table(plist, p=plist, acc=accs, m=[self.state[p]['exp_avg'] for p in plist],
                               v=[self.state[p]['exp_avg_sq'] for p in plist])
            tab['g'] = torch.zeros_like(tab['p'])          # the captured gradients' addresses, filled after capture
            groups.append(dict(gi=gi, plist=plist, accs=accs, tab=tab))
        if not groups:
            raise N.EffdetNativeError('FusedClipAdamW: none of its parameters receives a gradient')
        dev = groups[0]['plist'][0].device
        lrs = [float(g['lr']) for g in self.param_groups]
        self._graph = dict(
            groups=groups, frozen=self._frozen(), lr_host=lrs, update_host=0, src=None,
            step=torch.tensor(steps, dtype=torch.int64, device=dev),
            lr=torch.tensor(lrs, dtype=torch.float32, device=dev),
            update=torch.zeros((1,), dtype=torch.int32, device=dev),
            gate=torch.zeros((1,), dtype=torch.int32, device=dev),
            ticket=torch.zeros((1,), dtype=torch.int32, device=dev),
            norm_sq=torch.zeros((1,), dtype=torch.float32, device=dev))

    def _graph_launch(self, grads, loss):
        """Inside capture: accumulate this micro-step's gradients (grads: parameter -> gradient tensor) unless the
        loss is zero, then the gated clip + AdamW over the accumulators."""
        G = self._graph
        src = []
        for gr in G['groups']:
            gs = [grads.get(p) for p in gr['plist']]
            if any(g is None for g in gs):
                raise N.EffdetNativeError('FusedClipAdamW: a parameter that received a gradient while warming up '
                                          'received none during capture')
            for g in gs:
                if g.dtype != torch.float32 or not g.is_contiguous():
                    raise N.EffdetNativeError('FusedClipAdamW needs contiguous float32 gradients')
            src.append(gs)
        bound = {id(p) for gr in G['groups'] for p in gr['plist']}
        if any(id(p) not in bound and g is not None for p, g in grads.items()):
            raise N.EffdetNativeError('FusedClipAdamW: a parameter received a gradient during capture but none while '
                                      'warming up')
        G['src'] = src
        dev_t = G['step']
        for gr in G['groups']:
            t = gr['tab']
            N.call('effdet_multi_accumulate', dev_t, t['acc'].data_ptr(), t['g'].data_ptr(), t['numels'].data_ptr(),
                   t['ct'].data_ptr(), t['co'].data_ptr(), t['nchunks'], _CHUNK, loss.data_ptr(),
                   G['update'].data_ptr(), G['gate'].data_ptr())
        G['norm_sq'].zero_()
        for gr in G['groups']:
            t = gr['tab']
            N.call('effdet_multi_sumsq', dev_t, t['acc'].data_ptr(), t['numels'].data_ptr(), t['ct'].data_ptr(),
                   t['co'].data_ptr(), t['nchunks'], _CHUNK, G['norm_sq'].data_ptr())
        for gr in G['groups']:
            t, group = gr['tab'], self.param_groups[gr['gi']]
            b1, b2 = group['betas']
            N.call('effdet_multi_clip_adamw_dev', dev_t, t['p'].data_ptr(), t['acc'].data_ptr(), t['m'].data_ptr(),
                   t['v'].data_ptr(), t['numels'].data_ptr(), t['ct'].data_ptr(), t['co'].data_ptr(), t['nchunks'],
                   _CHUNK, G['norm_sq'].data_ptr(), float(group['max_norm'] or 0.0),
                   G['lr'][gr['gi']].data_ptr(), G['step'][gr['gi']].data_ptr(), G['gate'].data_ptr(),
                   G['ticket'].data_ptr(), float(b1), float(b2), float(group['eps']), float(group['weight_decay']))

    def _graph_captured(self):
        """After capture: the gradient tables get the captured gradients' addresses (the kernels read them at replay
        time), and p.grad becomes the accumulator."""
        G = self._graph
        for gr, gs in zip(G['groups'], G['src']):
            ptrs = np.array([g.data_ptr() for g in gs], dtype=np.uint64).view(np.int64)
            gr['tab']['g'].copy_(torch.from_numpy(ptrs))
            for p, a in zip(gr['plist'], gr['accs']):
                p.grad = a
        self.last_norm_sq = G['norm_sq']

    def _graph_prepare(self, update):
        """Before a replay: refuse changed hyperparameters, write the update flag and changed learning rates into
        their device scalars (launches on the current stream, no synchronisation)."""
        G = self._graph
        frozen = self._frozen()
        if frozen != G['frozen']:
            raise N.EffdetNativeError(
                'FusedClipAdamW: betas / eps / weight_decay / max_norm changed from %r at capture to %r; they are '
                'fixed in the CUDA graph, build a new GraphedTrainStep' % (G['frozen'], frozen))
        flag = 1 if update else 0
        if flag != G['update_host']:
            G['update'].fill_(flag)
            G['update_host'] = flag
        for gi, group in enumerate(self.param_groups):
            lr = float(group['lr'])
            if lr != G['lr_host'][gi]:
                G['lr'][gi].fill_(lr)
                G['lr_host'][gi] = lr

    def _sync_steps(self):
        steps = self._graph['step'].tolist()                 # the one device read
        for gr in self._graph['groups']:
            for p in gr['plist']:
                self.state[p]['step'] = steps[gr['gi']]

    def state_dict(self):
        if self._graph is not None:
            self._sync_steps()
        return super().state_dict()

    def load_state_dict(self, state_dict):
        if self._graph is not None:
            raise N.EffdetNativeError('FusedClipAdamW is bound to a GraphedTrainStep: load the optimizer state before '
                                      'building the graphed step')
        return super().load_state_dict(state_dict)

    def zero_grad(self, set_to_none=True):
        if self._graph is None:
            return super().zero_grad(set_to_none)
        torch._foreach_zero_([a for gr in self._graph['groups'] for a in gr['accs']])
