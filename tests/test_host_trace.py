"""Host-logic test of the nn.Module mirror WITHOUT a GPU: the C-ABI call layer (`_native.call/f32/ptr`) is
replaced by a recorder, a full EfficientDet-D0 training step (forward + backward) is driven through the real
autograd Functions on CPU tensors (values are garbage -- nothing is computed), and the recorded sequence of
entry-point calls is checked for

  * every call naming a declared entry point with the declared number of arguments,
  * every buffer handed to the dense-conv / weight-gradient entry points being large enough for the geometry
    in its argument struct (batch strides included -- the head writes straight into the concatenated
    [B, 49104, K] prediction buffers),
  * the per-class call counts of one steady-state step being exactly the ones the bench recorded
    (bench.py --full-breakdown `kernel_breakdown`, stored in tests/golden/d0_bench_launches.json).

This is a test of the product's HOST code; the oracle is used only to make the state dict.
"""
import bisect
import collections
import ctypes
import json
import os

import pytest
import torch

import effdet_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Recorder:
    def __init__(self):
        self.calls = []
        self.bases = []            # sorted base addresses of registered buffers
        self.size = {}             # base -> bytes available from base to the end of its storage

    def _register(self, t):
        st = t.untyped_storage()
        base = t.data_ptr()
        avail = st.nbytes() - (base - st.data_ptr())
        lo = bisect.bisect_left(self.bases, base)
        hi = bisect.bisect_left(self.bases, base + avail)
        for b in self.bases[lo:hi]:                     # stale registrations of memory the allocator re-used
            del self.size[b]
        del self.bases[lo:hi]
        self.bases.insert(lo, base)
        self.size[base] = avail
        return base

    def f32(self, t, name='tensor'):
        if t is None:
            return None
        assert t.dtype == torch.float32, name
        assert t.is_contiguous(), name
        return self._register(t)

    def ptr(self, t):
        return None if t is None else self._register(t)

    def avail(self, p):
        """bytes between pointer p and the end of the registered buffer containing it"""
        i = bisect.bisect_right(self.bases, p) - 1
        assert i >= 0, 'pointer %x was never handed out by f32()/ptr()' % p
        base = self.bases[i]
        assert p < base + self.size[base], 'pointer %x is outside every registered buffer' % p
        return base + self.size[base] - p

    def call(self, name, dev_tensor, *args, nbytes=0, flops=0):
        snap = []
        for a in args:
            if isinstance(a, ctypes.Array):
                snap.append([_struct_dict(a[i]) for i in range(len(a))])
            elif isinstance(a, ctypes.Structure):
                snap.append(_struct_dict(a))
            else:
                snap.append(a)
        self.calls.append((name, snap))
        self.check(name, snap)

    # ---- geometry checks -------------------------------------------------------------------------
    def need(self, p, floats, what):
        if p is None or floats <= 0:
            return
        assert self.avail(p) >= 4 * floats, '%s: buffer too small (%d < %d bytes)' % (what, self.avail(p), 4 * floats)

    def check(self, name, snap):
        if name in ('effdet_conv2d', 'effdet_conv2d_multi'):
            levels = snap[0] if isinstance(snap[0], list) else [snap[0]]
            if name == 'effdet_conv2d_multi':
                assert snap[1] == len(levels) and 1 <= len(levels) <= 8
            for a in levels:
                px, kk = a['H'] * a['W'], a['ksize'] ** 2
                assert a['ksize'] in (1, 3) and a['Cin'] % 4 == 0 and a['Cout'] % 4 == 0, a
                self.need(a['x'], (a['B'] - 1) * a['x_bstride'] + px * a['Cin'], name + ' x')
                assert (a['x'] is None) == (a['x_planes'] is not None)
                if a['x_planes'] is not None:             # bf16 hi/lo planes [2][B*H*W][Cin] = B*H*W*Cin floats' worth of bytes
                    assert a['ksize'] == 1 and a['Cin'] % 8 == 0 and a['in_scale'] is None and a['a_scale'] is None
                    self.need(a['x_planes'], a['B'] * px * a['Cin'], name + ' x_planes')
                self.need(a['y'], (a['B'] - 1) * a['y_bstride'] + px * a['Cout'], name + ' y')
                self.need(a['z'], a['B'] * px * a['Cout'], name + ' z')
                self.need(a['w'], kk * a['Cin'] * a['Cout'], name + ' w')
                for f in ('bias', 'scale', 'shift'):
                    self.need(a[f], a['Cout'], name + ' ' + f)
                self.need(a['a_scale'], a['B'] * a['Cin'], name + ' a_scale')
                self.need(a['in_scale'], a['Cin'], name + ' in_scale'); self.need(a['in_shift'], a['Cin'], name + ' in_shift')
                assert (a['in_scale'] is None) == (a['in_shift'] is None) and (a['in_scale'] is None or a['ksize'] == 1)
                self.need(a['row_scale'], a['B'], name + ' row_scale')
                self.need(a['residual'], (a['B'] - 1) * a['r_bstride'] + px * a['Cout'], name + ' residual')
                self.need(a['mask_src'], (a['B'] - 1) * a['m_bstride'] + px * a['Cout'], name + ' mask_src')
                assert a['x_bstride'] >= px * a['Cin'] and a['y_bstride'] >= px * a['Cout'], a
        elif name in ('effdet_conv2d_wgrad', 'effdet_conv2d_wgrad_multi'):
            levels = snap[0] if isinstance(snap[0], list) else [snap[0]]
            for a in levels:
                px, kk = a['H'] * a['W'], a['ksize'] ** 2
                self.need(a['x'], (a['B'] - 1) * a['x_bstride'] + px * a['Cin'], name + ' x')
                self.need(a['dy'], (a['B'] - 1) * a['dy_bstride'] + px * a['Cout'], name + ' dy')
                assert (a['dy'] is None) == (a['dy_planes'] is not None) and (a['x'] is None) == (a['x_planes'] is not None)
                pitch = lambda c: (c + 7) // 8 * 8                                       # noqa: E731
                if a['dy_planes'] is not None:                 # bf16 hi/lo planes [2][B*H*W][pitch]: 4 bytes per element
                    assert a['precision'] == 1 and a['dbias'] is None
                    self.need(a['dy_planes'], a['B'] * px * pitch(a['Cout']), name + ' dy_planes')
                if a['x_planes'] is not None:
                    assert a['precision'] == 1 and a['a_scale'] is None and a['in_scale'] is None
                    self.need(a['x_planes'], a['B'] * px * pitch(a['Cin']), name + ' x_planes')
                self.need(a['dw'], kk * a['Cin'] * a['Cout'], name + ' dw')
                self.need(a['dbias'], a['Cout'], name + ' dbias')
                self.need(a['a_scale'], a['B'] * a['Cin'], name + ' a_scale')
                self.need(a['in_scale'], a['Cin'], name + ' in_scale'); self.need(a['in_shift'], a['Cin'], name + ' in_shift')
                assert (a['ws_x'] is None) == (a['precision'] == 0 or a['x_planes'] is not None)
                assert (a['ws_dy'] is None) == (a['precision'] == 0 or a['dy_planes'] is not None)
        elif name == 'effdet_conv_planes_multi':
            levels = snap[0]
            assert snap[1] == len(levels) and 1 <= len(levels) <= 8
            pitch = lambda c: (c + 7) // 8 * 8                                           # noqa: E731
            for a in levels:
                px = a['H'] * a['W']
                assert a['ksize'] in (1, 3) and a['Cin'] % 4 == 0 and a['Cout'] % 4 == 0 and a['w_tc'] is not None
                assert a['y'] is not None or a['y_planes'] is not None
                self.need(a['x_planes'], a['B'] * px * pitch(a['Cin']), name + ' x_planes')
                self.need(a['y_planes'], a['B'] * px * pitch(a['Cout']), name + ' y_planes')
                self.need(a['mask_planes'], a['B'] * px * pitch(a['Cout']), name + ' mask_planes')
                self.need(a['y'], (a['B'] - 1) * a['y_bstride'] + px * a['Cout'], name + ' y')
                self.need(a['residual'], (a['B'] - 1) * a['r_bstride'] + px * a['Cout'], name + ' residual')
                self.need(a['bias'], a['Cout'], name + ' bias'); self.need(a['colsum'], a['Cout'], name + ' colsum')
        elif name == 'effdet_to_planes':
            x, x_bs, prob, p_bs, planes, colsum, B, HW, C = snap
            self.need(x, (B - 1) * x_bs + HW * C, 'to_planes x'); self.need(prob, (B - 1) * p_bs + HW * C, 'to_planes prob')
            self.need(planes, B * HW * ((C + 7) // 8 * 8), 'to_planes planes'); self.need(colsum, C, 'to_planes colsum')
        elif name in ('effdet_dwconv_fwd_fused', 'effdet_dwconv_bwd_fused'):
            a = snap[0]
            B, H, W, C, k, stride, Ho, Wo = (a[f] for f in ('B', 'H', 'W', 'C', 'k', 'stride', 'Ho', 'Wo'))
            assert (k, stride) in ((3, 1), (3, 2), (5, 1), (5, 2))
            # the reference's STATIC pads (models/utils.py:126-155; SURVEY.md 8(a) row B3) are compiled into the kernels
            assert (a['pad_t'], a['pad_l']) == {(3, 1): (1, 1), (3, 2): (0, 0), (5, 1): (2, 2), (5, 2): (1, 1)}[(k, stride)]
            total = {(3, 1): 2, (3, 2): 1, (5, 1): 4, (5, 2): 3}[(k, stride)]
            assert Ho == (H + total - k) // stride + 1 and Wo == (W + total - k) // stride + 1 and C % 4 == 0
            big, small = B * H * W * C, B * Ho * Wo * C
            if name == 'effdet_dwconv_fwd_fused':
                self.need(a['x'], big, 'dwf x'); self.need(a['z'], small, 'dwf z'); self.need(a['w_kkc'], k * k * C, 'dwf w')
                for f in ('in_scale', 'in_shift', 'scale', 'shift'):
                    self.need(a[f], C, 'dwf ' + f)
                self.need(a['se_sum'], B * C, 'dwf se_sum')
                assert (a['in_scale'] is None) == (a['in_shift'] is None) and abs(a['se_alpha'] * Ho * Wo - 1) < 1e-5
            else:
                self.need(a['dq'], small, 'dwb dq'); self.need(a['z1'], small, 'dwb z1')
                self.need(a['x'], big, 'dwb x'); self.need(a['dx'], big, 'dwb dx')
                assert (a['dx'] is None) == (a['dx_planes'] is not None)
                if a['dx_planes'] is not None:
                    assert C % 8 == 0 and a['scale0'] is not None          # only the expand-conv gradient takes this form
                    self.need(a['dx_planes'], big, 'dwb dx_planes')
                self.need(a['gate'], B * C, 'dwb gate'); self.need(a['dmean'], B * C, 'dwb dmean')
                self.need(a['w_kkc'], k * k * C, 'dwb w'); self.need(a['dw'], k * k * C, 'dwb dw')
                for f in ('scale1', 'shift1', 'mean1', 'rstd1', 'dgamma1', 'dbeta1'):
                    assert a[f] is not None
                    self.need(a[f], C, 'dwb ' + f)
                bn0 = [a[f] is not None for f in ('scale0', 'shift0', 'mean0', 'rstd0', 'dgamma0', 'dbeta0')]
                assert all(bn0) or not any(bn0)
                for f in ('scale0', 'shift0', 'mean0', 'rstd0', 'dgamma0', 'dbeta0'):
                    self.need(a[f], C, 'dwb ' + f)
                assert abs(a['inv_hw'] * Ho * Wo - 1) < 1e-5
        elif name == 'effdet_spatial_reduce_act':
            a, z, scale, shift, out, alpha, B, HW, C = snap
            self.need(a, B * HW * C, 'reduce a'); self.need(z, B * HW * C, 'reduce z'); self.need(out, B * C, 'reduce out')
            self.need(scale, C, 'reduce scale'); self.need(shift, C, 'reduce shift')
        elif name == 'effdet_stem_fwd':
            x, w, scale, shift, z, y, B, H, W, C0 = snap
            assert H % 2 == 0 and W % 2 == 0
            self.need(x, B * 3 * H * W, 'stem x'); self.need(w, C0 * 27, 'stem w')
            self.need(scale, C0, 'stem scale'); self.need(shift, C0, 'stem shift')
            self.need(z, B * (H // 2) * (W // 2) * C0, 'stem z'); self.need(y, B * (H // 2) * (W // 2) * C0, 'stem y')
        elif name == 'effdet_stem_wgrad':
            x, dz, dw, B, H, W, C0 = snap
            self.need(x, B * 3 * H * W, 'stem x'); self.need(dz, B * (H // 2) * (W // 2) * C0, 'stem dz')
            self.need(dw, C0 * 27, 'stem dw')
        elif name == 'effdet_se_gate_fwd':
            mean, w1, b1, w2, b2, s_pre, gate, B, C, S = snap
            assert S >= 1
            for p_, n_, w_ in ((mean, B * C, 'mean'), (w1, S * C, 'w1'), (b1, S, 'b1'), (w2, C * S, 'w2'), (b2, C, 'b2'),
                               (s_pre, B * S, 's_pre'), (gate, B * C, 'gate')):
                self.need(p_, n_, 'se_gate_fwd ' + w_)
        elif name == 'effdet_se_gate_bwd':
            dgate, mean, s_pre, gate, w1, w2, dmean, dw1, db1, dw2, db2, ws, B, C, S = snap
            self.need(ws, B * (C + S), 'se_gate_bwd ws')
            for p_, n_, w_ in ((dgate, B * C, 'dgate'), (mean, B * C, 'mean'), (s_pre, B * S, 's_pre'), (gate, B * C, 'gate'),
                               (w1, S * C, 'w1'), (w2, C * S, 'w2'), (dmean, B * C, 'dmean'), (dw1, S * C, 'dw1'),
                               (db1, S, 'db1'), (dw2, C * S, 'dw2'), (db2, C, 'db2')):
                self.need(p_, n_, 'se_gate_bwd ' + w_)
        elif name == 'effdet_bnact_bwd':
            a = snap[0]
            n = a['B'] * a['HW'] * a['C']
            for f in ('dy', 'z', 'dz'):
                self.need(a[f], n, 'bnact_bwd ' + f)
            for f in ('scale', 'shift', 'mean', 'rstd', 'dgamma', 'dbeta'):
                self.need(a[f], a['C'], 'bnact_bwd ' + f)
            self.need(a['row_scale'], a['B'], 'bnact_bwd row_scale')
            self.need(a['gate'], a['B'] * a['C'], 'bnact_bwd gate')
            self.need(a['dmean'], a['B'] * a['C'], 'bnact_bwd dmean')
            assert a['dy'] is not None and a['z'] is not None and a['dz'] is not None
        elif name in ('effdet_add', 'effdet_relu_bwd', 'effdet_sigmoid_bwd'):
            for p_ in snap[:3]:
                self.need(p_, snap[3], name)
        elif name == 'effdet_bn_fold':
            gamma, beta, mean, var, eps, scale, shift, rstd, C = snap
            assert abs(eps - 1e-3) < 1e-9                     # models/utils.py:273-274
            for p_ in (gamma, beta, mean, var, scale, shift, rstd):
                self.need(p_, C, 'bn_fold')
        elif name in ('effdet_focal_loss_fwd', 'effdet_focal_loss_bwd'):
            B, A, K, G = snap[-6:-2]
            assert (snap[-2], snap[-1]) == (0.25, 2.0)        # models/losses.py:33-34
            self.need(snap[0], B * A * K, 'focal cls'); self.need(snap[1], B * A * 4, 'focal reg')
            self.need(snap[2], A * 4, 'focal anchors'); self.need(snap[3], B * G * 5, 'focal annots')
            if name == 'effdet_focal_loss_bwd':
                self.need(snap[7], B * A * K, 'focal dcls'); self.need(snap[8], B * A * 4, 'focal dreg')


def _struct_dict(s):
    return {f[0]: getattr(s, f[0]) for f in s._fields_}


def _label(name, snap):
    """same class key as _native.Profiler.table()"""
    key = name.replace('effdet_', '')
    if name in ('effdet_conv2d', 'effdet_conv2d_wgrad'):
        a = snap[0]
        key += ' k%d %d->%d' % (a['ksize'], a['Cin'], a['Cout'])
    elif name in ('effdet_conv2d_multi', 'effdet_conv2d_wgrad_multi', 'effdet_conv_planes_multi'):
        a = snap[0][0]
        key += ' k%d %d->%d' % (a['ksize'], a['Cin'], a['Cout'])
    return key


@pytest.fixture()
def traced(monkeypatch):
    import __graft_entry__ as entry
    entry.build()                                    # effdet_conv_tc_kpad() is a host function of the real library
    from models import _native as N
    from models import _ops
    rec = Recorder()
    monkeypatch.setattr(N, 'f32', rec.f32)
    monkeypatch.setattr(N, 'ptr', rec.ptr)
    monkeypatch.setattr(N, 'call', rec.call)
    monkeypatch.setattr(_ops, 'check_cuda_f32', lambda x, what: None)
    monkeypatch.setattr(_ops, '_cache', {})
    return rec, N


def test_train_step_call_trace_matches_the_gpu_profile(traced):
    rec, N = traced
    from models import EfficientDet
    prof = json.load(open(os.path.join(REPO, 'tests', 'golden', 'd0_bench_launches.json')))
    assert prof['workload'].startswith('EfficientDet-D0')
    cfg = O.make_config('efficientdet-d0', 80, 64, 2)
    m = EfficientDet(num_classes=80, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=0))
    m.train()
    m.is_training = True
    m.freeze_bn()
    # the bench geometry (bs 32, 512x512): path decisions that depend on the map sizes (planes-based head, TMA pixel
    # boxes, small-map depthwise tiles) are then the ones the GPU run took; nothing is computed, torch.empty() of the
    # multi-GB activations only reserves address space
    images, ann = O.synthetic_batch(32, size=512, num_classes=80, seed=3)

    def step():
        for p in m.parameters():
            p.grad = None
        cl, rl = m([images, ann])
        assert tuple(cl.shape) == (1,) and tuple(rl.shape) == (1,)
        (cl.mean() + rl.mean()).backward()

    step()                                            # fills the parameter-derived caches (packs, folded BN)
    first = len(rec.calls)
    step()
    steady = rec.calls[first:]
    assert first > len(steady) > 300                  # the first step also packs weights and folds BN
    for name, snap in rec.calls:
        assert name in N.SIGNATURES, name
        assert len(snap) == len(N.SIGNATURES[name]) - 2, name          # (device, stream) are appended by call()
    got = collections.Counter(_label(n, s) for n, s in steady)
    want = prof['launches_per_step']
    assert dict(got) == want
    # every parameter that the reference trains received a gradient buffer of its own shape
    dead = [n for n, p in m.named_parameters() if p.grad is None]
    assert len(dead) == 5 and all(n.startswith('backbone.') for n in dead), dead
    for n, p in m.named_parameters():
        if p.grad is not None:
            assert p.grad.shape == p.shape and p.grad.dtype == torch.float32, n


@pytest.mark.parametrize('net,W,D,size', [('efficientdet-d2', 112, 4, 256), ('efficientdet-d4', 224, 6, 384)])
def test_scaled_variants_issue_consistent_geometry(traced, net, W, D, size):
    """the same buffer-extent checks (done inside Recorder.call) over the wider / deeper family members, plus the
    launch count formula: everything scales with (#MBConv blocks, D_bifpn), nothing with image size or batch"""
    rec, N = traced
    from models import EfficientDet
    cfg = O.make_config(net, 20, W, D)
    m = EfficientDet(num_classes=20, network=net, D_bifpn=D, W_bifpn=W, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=1))
    m.train()
    m.is_training = True
    m.freeze_bn()
    counts = []
    for B, s in ((1, size), (2, size - 128)):          # both multiples of 128, as the pyramid needs
        images, ann = O.synthetic_batch(B, size=s, num_classes=20, seed=4)
        for _ in range(2):
            for p in m.parameters():
                p.grad = None
            start = len(rec.calls)
            cl, rl = m([images, ann])
            (cl.mean() + rl.mean()).backward()
        counts.append(collections.Counter(n for n, _ in rec.calls[start:]))
    assert counts[0] == counts[1]
    c = counts[0]
    nblocks = len(cfg['blocks'])
    assert c['effdet_dwconv_fwd_fused'] == nblocks and c['effdet_dwconv_bwd_fused'] == nblocks
    assert c['effdet_spatial_reduce_act'] == nblocks and c['effdet_se_gate_bwd'] == nblocks
    assert c['effdet_bnact_bwd'] == nblocks + 1          # BN2 of every block + the stem; BN0/BN1 are fused away
    assert c['effdet_bifpn_fuse_fwd'] == 8 * D and c['effdet_bifpn_fuse_bwd'] == 8 * D
    assert c['effdet_focal_loss_fwd'] == 1 and c['effdet_focal_loss_bwd'] == 1 and c['effdet_stem_wgrad'] == 1


def test_second_backward_is_refused_with_a_clear_message(traced):
    """the fused nodes release their saved activations in the first backward; a retained graph must fail loudly, not with a
    TypeError on None (ADVICE round 1) -- and class counts that are not multiples of 4 go through the padded head"""
    rec, N = traced
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', 3, 64, 2)
    m = EfficientDet(num_classes=3, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=2))
    m.train()
    m.is_training = True
    m.freeze_bn()
    images, ann = O.synthetic_batch(1, size=128, num_classes=3, seed=5)
    cl, rl = m([images, ann])
    loss = cl.mean() + rl.mean()
    loss.backward(retain_graph=True)
    assert tuple(m.bbox_head.retina_cls.weight.grad.shape) == (27, 256, 3, 3)      # 9 anchors x 3 classes, unpadded
    with pytest.raises(N.EffdetNativeError, match='second time'):
        loss.backward()


def test_non_halving_pyramid_is_refused(traced):
    """192 = 1.5 * 128: P6 is 3x3 and P7 2x2 -- the reference dies with a shape mismatch inside BiFPNModule.forward
    (models/bifpn.py:188-201); the drop-in must refuse too instead of letting the fusion kernel index out of range"""
    rec, N = traced
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=2))
    images, ann = O.synthetic_batch(1, size=192, num_classes=20, seed=5)
    with pytest.raises(N.EffdetNativeError, match='halve exactly'):
        m([images, ann])


def test_parameter_updates_invalidate_the_packed_weight_caches(traced, monkeypatch):
    """packed conv weights / folded BN are cached per parameter and keyed on (Tensor._version, data_ptr): a step
    without an update re-uses them, an in-place update of ONE weight re-packs only that weight, and the fused
    optimizer (whose kernel writes through raw pointers) must bump the versions itself so that EVERYTHING is
    re-derived -- otherwise training would silently keep convolving with the initial weights"""
    rec, N = traced
    from models import EfficientDet
    from models import fused_optim
    monkeypatch.setattr(fused_optim, '_check_param', lambda p: None)
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=2))
    m.train()
    m.is_training = True
    m.freeze_bn()
    images, ann = O.synthetic_batch(1, size=128, num_classes=20, seed=5)
    derived = ('effdet_pack_conv_weight', 'effdet_pack_conv_weight_tc', 'effdet_pack_dw_weight', 'effdet_bn_fold')

    def step(zero=True):
        if zero:
            for p in m.parameters():
                p.grad = None
        start = len(rec.calls)
        cl, rl = m([images, ann])
        (cl.mean() + rl.mean()).backward()
        return collections.Counter(n for n, _ in rec.calls[start:] if n in derived)

    cold = step()
    # 31 backbone 1x1 (15 expand + 16 project) + 5 laterals + 16 BiFPN + 10 head convs; stem + 15 + 16 + 16 BatchNorms
    assert cold == {'effdet_pack_conv_weight': 62, 'effdet_pack_conv_weight_tc': 62, 'effdet_pack_dw_weight': 16,
                    'effdet_bn_fold': 48}
    assert sum(step().values()) == 0                                   # warm: nothing re-derived
    with torch.no_grad():
        m.bbox_head.retina_cls.weight.mul_(1.0)                        # in-place update of one parameter
    again = step()
    assert again == {'effdet_pack_conv_weight': 1, 'effdet_pack_conv_weight_tc': 1}
    with torch.no_grad():
        m.backbone._bn0.weight.add_(0.0)
    assert step() == {'effdet_bn_fold': 1}
    # torch's own optimizer updates in place -> everything with a gradient is re-derived
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    opt.step()
    after_torch = step()
    # the fused optimizer must have the same effect
    fused = fused_optim.FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1)
    v0 = m.bbox_head.retina_cls.weight._version
    g0 = m.bbox_head.retina_cls.weight.grad._version
    fused.step()
    assert m.bbox_head.retina_cls.weight._version > v0 and m.bbox_head.retina_cls.weight.grad._version > g0
    names = [n for n, _ in rec.calls[-2:]]
    assert names == ['effdet_multi_sumsq', 'effdet_multi_clip_adamw']
    after_fused = step()
    assert after_fused == after_torch
    assert after_fused == cold                                          # every live parameter was re-derived


def test_batch_statistics_batchnorm_is_refused(traced):
    """model.train() WITHOUT freeze_bn() puts BatchNorm in batch-statistics mode: the reference would then normalise
    with batch statistics, the kernels only implement the frozen BatchNorm -> refuse instead of diverging silently"""
    rec, N = traced
    from models import EfficientDet
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    images, ann = O.synthetic_batch(1, size=128, num_classes=20, seed=5)
    m([images, ann])                                  # as constructed: BN already frozen (models/efficientdet.py:55)
    m.train()
    with pytest.raises(N.EffdetNativeError, match='freeze_bn'):
        m([images, ann])
    m.freeze_bn()
    m([images, ann])
