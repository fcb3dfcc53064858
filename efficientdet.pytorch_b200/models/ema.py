"""Exponential moving average of the weights, the EfficientDet paper's "exponential moving average with decay 0.9998"
(Tan et al. 2020, section 5.1): a shadow copy of the model whose every floating-point state entry follows

    d = min(decay, (1 + k) / (10 + k))   (ramp=True; d = decay otherwise),   e = e - (1 - d) * (e - s)

at update number k, as TF's ExponentialMovingAverage(decay, num_updates) does in google/automl.  One multi-tensor
launch (effdet_multi_ema) updates all of it; the counter k lives on the device.

    ema = ModelEma(model)                              # model: EfficientDet or its DDP wrapper, on the GPU
    loss.backward(); opt.step(); ema.update(model)     # eager loops: one launch per call
    step = GraphedTrainStep(model, ..., optimizer=opt, ema=ema)   # graphed: the launch is part of every replay
    ema.module.detect_batch(images); evaluate(generator, ema.module)

Eager `update` and every GraphedTrainStep call bump the versions of the averaged tensors, so the packed-weight and
folded-BatchNorm caches of models/_ops.py are rebuilt from the new values before ema.module next runs.
"""
import copy
import weakref

import torch

from . import _native as N
from .efficientdet import EfficientDet
from .fused_optim import _CHUNK, _chunk_table


def _unwrap(model):
    return model.module if isinstance(model, torch.nn.parallel.DistributedDataParallel) else model


class ModelEma:
    def __init__(self, model, decay=0.9998, ramp=True):
        model = _unwrap(model)
        if not isinstance(model, EfficientDet):
            raise N.EffdetNativeError('ModelEma averages an EfficientDet (or its DDP wrapper), got %s'
                                      % type(model).__name__)
        decay = float(decay)
        if not 0.0 <= decay <= 1.0:
            raise N.EffdetNativeError('ModelEma: decay must lie in [0, 1], got %r' % decay)
        self.decay, self.ramp = decay, bool(ramp)
        src = model.state_dict()
        self._check(src, 'the model')
        module = copy.deepcopy(model)                    # same architecture and post-processing attributes
        for p in module.parameters():
            p.requires_grad_(False)
        module.eval()
        module.is_training = False
        self.module = module
        sd = module.state_dict()
        self._shapes = [(k, tuple(v.shape), v.is_floating_point()) for k, v in sd.items()]
        self._names = [k for k, v in sd.items() if v.is_floating_point()]
        self._avg = [sd[k] for k in self._names]
        dev = self._avg[0].device
        self.updates = torch.zeros((1,), dtype=torch.int64, device=dev)
        self._ticket = torch.zeros((1,), dtype=torch.int32, device=dev)
        self._src = None                                 # (weakref to the model, its state tensors)
        self._tables = {}

    @staticmethod
    def _check(sd, what):
        for k, v in sd.items():
            if not v.is_cuda:
                raise N.EffdetNativeError('ModelEma needs %s on a CUDA device (%s is on %s); there is no CPU path'
                                          % (what, k, v.device))
            if v.is_floating_point() and (v.dtype != torch.float32 or not v.is_contiguous()):
                raise N.EffdetNativeError('ModelEma needs contiguous float32 state in %s (%s: %s)' % (what, k, v.dtype))

    def _table(self, model):
        """the chunk tables from the model's floating-point state to the averaged tensors, refused when the model's
        state-dict schema differs from ema.module's.  The model's state tensors (parameters and buffers, as objects)
        are collected once per model, since state_dict() alone costs more host time than the update; the tables are
        cached per set of their addresses, so in-place moves of parameter data are followed."""
        model = _unwrap(model)
        if self._src is None or self._src[0]() is not model:
            sd = model.state_dict(keep_vars=True)
            if [(k, tuple(v.shape), v.is_floating_point()) for k, v in sd.items()] != self._shapes:
                raise N.EffdetNativeError('ModelEma: the model\'s state-dict keys or shapes differ from ema.module\'s')
            self._src = (weakref.ref(model), [sd[k] for k in self._names])
        src = self._src[1]
        key = tuple(t.data_ptr() for t in src)
        tab = self._tables.get(key)
        if tab is None:
            self._check(dict(zip(self._names, src)), 'the model')
            if src[0].device != self._avg[0].device:
                raise N.EffdetNativeError('ModelEma: the model is on %s, the average on %s'
                                          % (src[0].device, self._avg[0].device))
            tab = self._tables[key] = _chunk_table(self._avg, e=self._avg, s=src)
        return tab

    def _launch(self, tab, gate=None):
        """one effdet_multi_ema launch on the current stream; gate: the optimizer's device gate, or None"""
        N.call('effdet_multi_ema', self.updates, tab['e'].data_ptr(), tab['s'].data_ptr(), tab['numels'].data_ptr(),
               tab['ct'].data_ptr(), tab['co'].data_ptr(), tab['nchunks'], _CHUNK, self.decay, int(self.ramp),
               self.updates.data_ptr(), None if gate is None else gate.data_ptr(), self._ticket.data_ptr())

    def _bump_versions(self):
        # the kernel writes through raw pointers: the version-keyed caches of models/_ops.py must see a change
        torch.autograd.graph.increment_version(self._avg)

    @torch.no_grad()
    def update(self, model):
        """One update from the model's current state (call it after every optimizer step of an eager loop)."""
        self._launch(self._table(model))
        self._bump_versions()

    def state_dict(self):
        """{'module': ema.module's state dict (its live tensors, like nn.Module.state_dict), 'updates': k, 'decay',
        'ramp'}; reading k is the one device read"""
        return {'module': self.module.state_dict(), 'updates': int(self.updates.item()), 'decay': self.decay,
                'ramp': self.ramp}

    @torch.no_grad()
    def load_state_dict(self, state):
        """Copies the averaged state and the counter in place: a GraphedTrainStep built with this ModelEma keeps
        reading the same addresses.  decay and ramp must match this ModelEma's (they are fixed in captured graphs)."""
        if (float(state['decay']), bool(state['ramp'])) != (self.decay, self.ramp):
            raise N.EffdetNativeError('ModelEma: the state has decay=%r, ramp=%r, this ModelEma decay=%r, ramp=%r'
                                      % (state['decay'], state['ramp'], self.decay, self.ramp))
        src = state['module']
        if [(k, tuple(v.shape), v.is_floating_point()) for k, v in src.items()] != self._shapes:
            raise N.EffdetNativeError('ModelEma: the state\'s keys or shapes differ from ema.module\'s')
        for k, v in self.module.state_dict().items():
            v.copy_(src[k])
        self.updates.fill_(int(state['updates']))
        self._bump_versions()
