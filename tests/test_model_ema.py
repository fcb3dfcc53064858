"""Weight EMA (models/ema.py ModelEma, csrc/optim.cu effdet_multi_ema): the moving average of the weights that the
EfficientDet paper evaluates, updated eagerly or inside GraphedTrainStep's replay.

CPU: the entry point's refusals; tools/ema_oracle.py against a literal transcription of TF's assign_moving_average with
the num_updates ramp (bit for bit) and against timm's ModelEmaV2 formula (within 2 ulp); no CPU model.
GPU: the kernel against the oracle bit for bit (chunk edges, the ramp, the gate, the counter and its ticket); eager
updates after FusedClipAdamW steps; the graphed step with accumulation and a zero-loss batch in static, capacity and
raw mode; inference on the averaged weights after replays, with a stale-cache control; a checkpoint round trip; the
launch count; DDP on 2 GPUs."""
import io
import os
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O
from test_graphed_train_loop import _d0, _free_port
from test_raw_batches import _samples
from test_voc_eval import _Generator

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
import ema_oracle as E  # noqa: E402
import voc_eval_oracle as V  # noqa: E402

FAKE = 1 << 20                                               # aligned non-null "pointer"; never dereferenced
DECAY = 0.9998
# Two forward passes over the same weights differ in the last bits: dw_fwd_fused_kernel sums the squeeze-excite means
# with fp32 atomics.  Network outputs are compared at the bf16x3 tolerance.
TOL_FWD = 1e-3


def _dev():
    return torch.device('cuda:0')


def _bits(t):
    return np.ascontiguousarray(np.asarray(t, dtype=np.float32)).view(np.uint32)


def _same_bits(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _host(sd):
    """the floating-point entries of a state dict as float32 NumPy arrays"""
    return {k: v.detach().cpu().numpy().copy() for k, v in sd.items() if v.is_floating_point()}


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------

def test_multi_ema_refuses_bad_arguments():
    from models import _native
    _native.build()
    lib = _native.load()
    good = [FAKE] * 5 + [1, 64, DECAY, 1, FAKE, None, FAKE]
    for i in (0, 1, 2, 3, 4, 9, 11):                          # every table, the counter, the ticket
        args = list(good)
        args[i] = None
        assert lib.effdet_multi_ema(*args, 0, None) == -1, i
        assert 'multi_ema' in lib.effdet_last_error().decode(), i
    for i, bad in ((5, 0), (6, 0), (7, -0.1), (7, 1.5), (7, float('nan'))):
        args = list(good)
        args[i] = bad
        assert lib.effdet_multi_ema(*args, 0, None) == -1, (i, bad)
        assert 'multi_ema' in lib.effdet_last_error().decode(), (i, bad)
    assert 'decay' in lib.effdet_last_error().decode()


def _tf_ema_decay(decay, num_updates):
    """tensorflow/python/training/moving_averages.py, ExponentialMovingAverage.apply with num_updates"""
    return min(decay, (1.0 + num_updates) / (10.0 + num_updates))


def _tf_assign_moving_average(variable, value, decay):
    """moving_averages.assign_moving_average(variable, value, decay, zero_debias=False) on a float32 variable, with
    decay a Python float: decay = convert_to_tensor(1.0 - decay) cast to the variable's dtype, then
    variable.assign_sub((variable - value) * decay)"""
    decay = np.float32(1.0 - decay)
    update_delta = (variable - value) * decay
    return variable - update_delta


def _pairs(seed, n=200000):
    rng = np.random.default_rng(seed)
    mag = (10.0 ** rng.uniform(-6, 3, n)).astype(np.float32)
    e = (rng.standard_normal(n) * mag).astype(np.float32)
    s = np.where(rng.random(n) < 0.5, e * (1 + 1e-3 * rng.standard_normal(n)),             # a model near its average
                 rng.standard_normal(n) * mag).astype(np.float32)
    s[:100] = e[:100]                                         # equal entries (frozen BatchNorm) stay put
    return e, s


@pytest.mark.parametrize('k', [1, 2, 9, 10, 1000, 10 ** 6])
def test_oracle_equals_tf_assign_moving_average_and_timm_within_2_ulp(k):
    e, s = _pairs(k)
    want = _tf_assign_moving_average(e, s, _tf_ema_decay(DECAY, k))
    got = E.apply([e], [s], k, DECAY)[0]
    assert got.dtype == np.float32 and _same_bits(got, want)
    assert _same_bits(got[:100], e[:100])
    assert _same_bits(E.apply([e], [s], k, DECAY, ramp=False)[0], _tf_assign_moving_average(e, s, DECAY))
    d = _tf_ema_decay(DECAY, k)
    timm = np.float32(d) * e + np.float32(1.0 - d) * s          # timm ModelEmaV2: e * d + (1 - d) * s in fp32
    ulp = np.spacing(np.maximum(np.abs(e), np.abs(s)))
    worst = float(np.max(np.abs(got.astype(np.float64) - timm.astype(np.float64)) / ulp))
    print('k=%d: oracle vs timm ModelEmaV2 worst %.2f ulp' % (k, worst))
    assert worst <= 2.0


def test_cpu_model_is_refused():
    from models import EfficientDet, _native
    from models.ema import ModelEma
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64)
    with pytest.raises(_native.EffdetNativeError, match='CUDA'):
        ModelEma(m)
    with pytest.raises(_native.EffdetNativeError, match='EfficientDet'):
        ModelEma(torch.nn.Linear(2, 2))


# ------------------------------------------------------------------------------------------------------------------
# GPU, kernel level
# ------------------------------------------------------------------------------------------------------------------

SIZES = [1, 65535, 65536, 65537, 3 * 65536 + 5]


def _kernel_launch(ema, src, updates, ticket, ramp, gate):
    from models import _native as N
    from models.fused_optim import _CHUNK, _chunk_table
    tab = _chunk_table(ema, e=ema, s=src)
    assert tab['nchunks'] == 9                               # a multi-CTA grid with partial and single-element chunks
    N.call('effdet_multi_ema', updates, tab['e'].data_ptr(), tab['s'].data_ptr(), tab['numels'].data_ptr(),
           tab['ct'].data_ptr(), tab['co'].data_ptr(), tab['nchunks'], _CHUNK, DECAY, int(ramp), updates.data_ptr(),
           None if gate is None else gate.data_ptr(), ticket.data_ptr())


@pytest.mark.gpu
def test_kernel_equals_oracle_bit_for_bit():
    rng = np.random.default_rng(5)
    e0 = [rng.standard_normal(n).astype(np.float32) for n in SIZES]
    s0 = [(x + 0.05 * rng.standard_normal(x.size)).astype(np.float32) for x in e0]
    s0[4][:1000] = e0[4][:1000]
    dev = _dev()
    src = [torch.from_numpy(x).to(dev) for x in s0]
    ticket = torch.zeros((1,), dtype=torch.int32, device=dev)
    for ramp, k in ((True, 1), (True, 2), (True, 10), (True, 10 ** 6), (False, 7)):
        ema = [torch.from_numpy(x).to(dev) for x in e0]
        updates = torch.tensor([k - 1], dtype=torch.int64, device=dev)
        _kernel_launch(ema, src, updates, ticket, ramp, None)
        want = E.apply(e0, s0, k, DECAY, ramp)
        for n, got, w in zip(SIZES, ema, want):
            assert _same_bits(got.cpu().numpy(), w), (ramp, k, n)
        assert int(updates) == k and int(ticket) == 0, (ramp, k)

    ema = [torch.from_numpy(x).to(dev) for x in e0]
    updates = torch.tensor([4], dtype=torch.int64, device=dev)
    gate = torch.zeros((1,), dtype=torch.int32, device=dev)
    _kernel_launch(ema, src, updates, ticket, True, gate)      # gate 0: no byte, no count
    assert all(_same_bits(g.cpu().numpy(), x) for g, x in zip(ema, e0))
    assert int(updates) == 4 and int(ticket) == 0
    want = e0
    for i, g in enumerate((1, None, 1, None)):                # gate 1 and NULL: one update each, in stream order
        _kernel_launch(ema, src, updates, ticket, True, None if g is None else gate.fill_(g))
        want = E.apply(want, s0, 5 + i, DECAY)
        assert int(updates) == 5 + i and int(ticket) == 0, i
        assert all(_same_bits(t.cpu().numpy(), w) for t, w in zip(ema, want)), i


# ------------------------------------------------------------------------------------------------------------------
# GPU, whole model
# ------------------------------------------------------------------------------------------------------------------

CFG = dict(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64)


def _model(seed=43):
    return _d0(O.init_state_dict(O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2), seed=seed))


def _batches(n, zero_at=(), size=128, B=2, seed=60):
    out = []
    for i in range(n):
        images, ann = O.synthetic_batch(B, size=size, num_classes=20, seed=seed + i)
        if i in zero_at:
            ann[:] = -1                                       # no annotations: the loss is exactly 0
        out.append((images.to(_dev()), ann.to(_dev())))
    return out


def _opt_step(opt):
    return int(next(iter(opt.state_dict()['state'].values()))['step'])


def _assert_ema(ema, want, what):
    got = _host(ema.module.state_dict())
    assert got.keys() == want.keys()
    bad = [k for k in want if not _same_bits(got[k], want[k])]
    assert not bad, '%s: %d tensors differ, first %s' % (what, len(bad), bad[:3])


@pytest.mark.gpu
def test_eager_updates_after_fused_steps_equal_oracle():
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    m = _model()
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    ema = ModelEma(m)
    assert not ema.module.training and not ema.module.is_training
    assert not any(p.requires_grad for p in ema.module.parameters())
    assert (ema.module.threshold, ema.module.nms, ema.module.class_nms) == (m.threshold, m.nms, m.class_nms)
    want = _host(ema.module.state_dict())
    assert all(_same_bits(want[k], v) for k, v in _host(m.state_dict()).items())
    for i, (images, ann) in enumerate(_batches(5)):
        opt.zero_grad()
        cl, rl = m([images, ann])
        (cl.mean() + rl.mean()).backward()
        opt.step()
        ema.update(m)
        want = E.apply(want, _host(m.state_dict()), i + 1, DECAY)
        _assert_ema(ema, want, 'update %d' % (i + 1))
    assert ema.state_dict()['updates'] == 5
    frozen = [k for k in want if 'running' in k]
    assert frozen and all(_same_bits(want[k], m.state_dict()[k].cpu().numpy()) for k in frozen)


def _raw_batches(n, zero_at, S=128, B=2):
    from models.pipeline import RawCollater
    col = RawCollater(S, pixel_scale=255)
    out = []
    for i in range(n):
        samples = _samples(70 + i, [(96, 128), (128, 80)][:B], [3, 2][:B])
        if i in zero_at:
            for s in samples:
                s['annot'][:, 4] = -1
        out.append(col(samples))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['static', 'capacity', 'raw'])
def test_graphed_step_with_accumulation_equals_oracle_at_update_boundaries(mode):
    """k = 2 over 6 micro-batches; batch 3 (an update boundary) has no annotations.  After every replay the EMA is the
    oracle applied at the real updates only, and its counter is the optimizer's step advance."""
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    k, zero_at = 2, (3,)
    m = _model(seed=44)
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    ema = ModelEma(m)
    want = _host(ema.module.state_dict())
    if mode == 'raw':
        batches = [(r,) for r in _raw_batches(6, zero_at)]
        step = GraphedTrainStep(m, batches[0][0], optimizer=opt, ema=ema, max_annotations=8)
    else:
        batches = _batches(6, zero_at, B=3 if mode == 'capacity' else 2)
        if mode == 'capacity':
            batches[2] = (batches[2][0][:2], batches[2][1][:2, :5])          # a short batch with fewer rows
            step = GraphedTrainStep(m, *batches[0], optimizer=opt, ema=ema, max_annotations=16)
        else:
            step = GraphedTrainStep(m, *batches[0], optimizer=opt, ema=ema)
    torch.cuda.synchronize()
    _assert_ema(ema, want, 'after building the step')
    assert int(ema.updates) == 0
    step0, n_upd = _opt_step(opt), 0
    opt.zero_grad()
    for idx, b in enumerate(batches):
        update = (idx + 1) % k == 0
        loss = float(step(*b, update=update))
        assert (loss == 0.0) == (idx in zero_at), (idx, loss)
        if update and loss != 0.0:
            n_upd += 1
            want = E.apply(want, _host(m.state_dict()), n_upd, DECAY)
        _assert_ema(ema, want, '%s replay %d' % (mode, idx))
        assert int(ema.updates) == n_upd == _opt_step(opt) - step0, idx
    assert n_upd == 2


def _fresh(sd, like):
    from models import EfficientDet
    f = EfficientDet(is_training=False, **CFG)
    f.load_state_dict(sd)                                    # strict: the reference's state-dict schema
    f = f.to(_dev()).eval()
    for a in ('threshold', 'iou_threshold', 'nms', 'soft_nms_sigma', 'class_nms', 'pre_nms_top_k'):
        setattr(f, a, getattr(like, a))
    return f


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / max(float(b.norm()), 1e-30))


def _trained_ema(seed, replays=3):
    """a graphed D0 step with ema=, built and replayed `replays` times at a learning rate that moves the weights;
    ema.module runs eagerly once between the build and the replays, so its caches hold the initial average"""
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    m = _model(seed=seed)
    m.threshold = 0.01
    opt = FusedClipAdamW(m.parameters(), lr=2e-3, max_norm=0.1)
    ema = ModelEma(m)
    batches = _batches(replays, seed=80)
    step = GraphedTrainStep(m, *batches[0], optimizer=opt, ema=ema)
    x = _batches(1, size=128, B=4, seed=90)[0][0]
    with torch.no_grad():
        ema.module._raw_predictions(x)
    for b in batches:
        step(*b)
    torch.cuda.synchronize()
    return ema, x


@pytest.mark.gpu
def test_averaged_weights_drive_inference_after_replays(monkeypatch):
    """ema.module(img), detect_batch, a GraphedDetect on ema.module and evaluate() against a fresh EfficientDet loaded
    with ema.module.state_dict(); the control, with the version bump removed, reads stale packed weights"""
    from models import evaluation
    from models.ema import ModelEma
    from models.graph_step import GraphedDetect
    ema, x = _trained_ema(seed=45)
    with torch.no_grad():                # every eager call on ema.module before anything (a model's construction,
        got = ema.module._raw_predictions(x)            # eval(), load_state_dict) drops the caches
        got_one = [ema.module(x[:1])]
        got_b = ema.module.detect_batch(x)
    fresh = _fresh(ema.module.state_dict(), ema.module)

    def rows(d):
        """one image's detections in an order that the forward's last-bit noise cannot change (near-tied scores
        may swap places): by class, then box corner"""
        s, c, b = (t.detach().double().cpu().numpy() for t in d)
        o = np.lexsort((np.round(b[:, 1], 2), np.round(b[:, 0], 2), c))
        return torch.from_numpy(s[o]), c[o], torch.from_numpy(b[o])

    def same_dets(a, b, what):
        assert len(a) == len(b), what
        for i, (da, db) in enumerate(zip(a, b)):
            assert da[0].numel() == db[0].numel(), (what, i)
            if db[0].numel():
                (sa, ca, ba), (sb, cb, bb) = rows(da), rows(db)
                assert np.array_equal(ca, cb), (what, i)
                assert _rel(sa, sb) < TOL_FWD and _rel(ba, bb) < TOL_FWD, (what, i)

    with torch.no_grad():
        ref = fresh._raw_predictions(x)
        errs = [_rel(got[i], ref[i]) for i in (0, 1)]
        print('raw predictions rel err cls %.2e reg %.2e' % tuple(errs))
        assert max(errs) < TOL_FWD
        same_dets(got_one, [fresh(x[:1])], 'model(img)')
        ref_b = fresh.detect_batch(x)
        assert sum(d[0].numel() for d in ref_b) > 0
        same_dets(got_b, ref_b, 'detect_batch')
    det = GraphedDetect(ema.module, x, max_candidates=None)
    same_dets(det.to_list(det(x)), ref_b, 'GraphedDetect')

    images = [x[i].permute(1, 2, 0).contiguous().cpu() for i in range(4)]
    gen = _Generator(images, [1.0] * 4, [np.zeros((0, 5))] * 4, 20)
    dets = V.get_detections(gen, fresh, score_threshold=0.01)
    anns = []
    for i in range(4):                   # ground truth on every other box of the model's own with a positive area
        rows = [[d[0], d[1], d[2], d[3], c] for c in range(20) for d in dets[i][c][::2] if d[2] > d[0] and d[3] > d[1]]
        anns.append(np.array(rows + [[1000, 1000, 1010, 1010, 5]], np.float64))
    gen = _Generator(images, [1.0] * 4, anns, 20)
    got_map, got_aps = evaluation.evaluate(gen, ema.module, score_threshold=0.01, batch_size=4)
    want_map, want_aps = evaluation.evaluate(gen, fresh, score_threshold=0.01, batch_size=4)
    n_pos = sum(len(a) - 1 for a in anns)
    print('evaluate: %d detections, %d ground-truth boxes of positive area, mAP %.6f (fresh) %.6f (ema.module)'
          % (sum(len(d[c]) for d in dets for c in range(20)), n_pos, want_map, got_map))
    assert n_pos > 0 and want_map > 0
    assert abs(got_map - want_map) < TOL_FWD
    assert all(abs(got_aps[c][0] - want_aps[c][0]) < TOL_FWD and got_aps[c][1] == want_aps[c][1] for c in want_aps)

    monkeypatch.setattr(ModelEma, '_bump_versions', lambda self: None)
    ema, x = _trained_ema(seed=45)
    with torch.no_grad():
        got = ema.module._raw_predictions(x)
        ref = _fresh(ema.module.state_dict(), ema.module)._raw_predictions(x)
    ctrl = [_rel(got[i], ref[i]) for i in (0, 1)]
    print('stale-cache control rel err cls %.2e reg %.2e' % tuple(ctrl))
    assert max(ctrl) > TOL_FWD


@pytest.mark.gpu
def test_checkpoint_round_trip_resumes_the_average():
    """ema.state_dict() after 3 graphed steps, loaded into a new ModelEma on a new graphed step (after it is built),
    then 3 more steps: the oracle continued from the saved state over the resumed run's own parameters"""
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    batches = _batches(6, seed=100)
    m = _model(seed=46)
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    ema = ModelEma(m)
    step = GraphedTrainStep(m, *batches[0], optimizer=opt, ema=ema)
    for b in batches[:3]:
        step(*b)
    buf = io.BytesIO()
    torch.save({'state_dict': m.state_dict(), 'optimizer': opt.state_dict(), 'ema': ema.state_dict()}, buf)
    del step
    buf.seek(0)
    ck = torch.load(buf, map_location='cpu')
    assert ck['ema']['updates'] == 3 and ck['ema']['decay'] == DECAY and ck['ema']['ramp'] is True
    ref_sd = O.init_state_dict(O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2), seed=1)
    assert [(k, tuple(v.shape)) for k, v in ck['ema']['module'].items()] == \
        [(k, tuple(v.shape)) for k, v in ref_sd.items()]
    _fresh(ck['ema']['module'], m)

    m2 = _d0(ck['state_dict'])
    opt2 = FusedClipAdamW(m2.parameters(), lr=1e-3, max_norm=0.1)
    opt2.load_state_dict(ck['optimizer'])
    ema2 = ModelEma(m2)
    step2 = GraphedTrainStep(m2, *batches[0], optimizer=opt2, ema=ema2)
    ema2.load_state_dict(ck['ema'])
    want = _host(ck['ema']['module'])
    _assert_ema(ema2, want, 'loaded')
    for i, b in enumerate(batches[3:]):
        step2(*b)
        want = E.apply(want, _host(m2.state_dict()), 4 + i, DECAY)
        _assert_ema(ema2, want, 'resumed step %d' % (4 + i))
    assert ema2.state_dict()['updates'] == 6
    with pytest.raises(RuntimeError, match='decay'):
        ModelEma(m2, decay=0.999).load_state_dict(ck['ema'])


@pytest.mark.gpu
def test_ema_adds_one_library_launch_and_needs_an_optimizer():
    from models import _native as N
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    images, ann = _batches(1)[0]
    counts = []
    for with_ema in (False, True):
        m = _model()
        opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
        step = GraphedTrainStep(m, images, ann, optimizer=opt, ema=ModelEma(m) if with_ema else None)
        counts.append(step.library_launches)
        del step
    assert counts[1] == counts[0] + 1, counts
    m = _model()
    with pytest.raises(N.EffdetNativeError, match='optimizer'):
        GraphedTrainStep(m, images, ann, ema=ModelEma(m))


def _ddp_worker(rank, world, port, out):
    os.environ['TORCH_NCCL_ASYNC_ERROR_HANDLING'] = '0'
    os.environ['NCCL_ASYNC_ERROR_HANDLING'] = '0'
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    for p in (os.path.join(os.path.dirname(HERE), 'oracle'), os.path.join(os.path.dirname(HERE), 'efficientdet.pytorch_b200')):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    from models import EfficientDet
    from models.ema import ModelEma
    from models.fused_optim import FusedClipAdamW
    from models.graph_step import GraphedTrainStep
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    sd = O.init_state_dict(O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2), seed=3)
    batches = [O.synthetic_batch(2 * world, size=128, num_classes=20, seed=s_) for s_ in (92, 93, 94)]
    lo, hi = rank * 2, (rank + 1) * 2
    m = EfficientDet(is_training=True, **CFG)
    m.load_state_dict(sd)
    m = m.to(dev)
    m.eval()
    m.is_training = True
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        net = torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], find_unused_parameters=True,
                                                        static_graph=True, gradient_as_bucket_view=True,
                                                        broadcast_buffers=False)
    torch.cuda.current_stream(dev).wait_stream(side)
    opt = FusedClipAdamW(m.parameters(), lr=1e-3, max_norm=0.1)
    ema = ModelEma(net)
    step = GraphedTrainStep(net, batches[0][0][lo:hi].to(dev), batches[0][1][lo:hi].to(dev), optimizer=opt, ema=ema)
    for images, ann in batches:
        step(images[lo:hi].to(dev), ann[lo:hi].to(dev))
    torch.cuda.synchronize()
    torch.save({'ema': {k: v.cpu() for k, v in ema.state_dict()['module'].items()}, 'updates': int(ema.updates)},
               os.path.join(out, 'r%d.pt' % rank))
    dist.barrier(device_ids=[rank])
    os._exit(0)                                                 # (NCCL teardown after a captured collective hangs)


@pytest.mark.gpu
@pytest.mark.timeout(600)
def test_ddp_ranks_average_the_same_weights(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_ddp_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp_path, 'r%d.pt' % r)) for r in (0, 1))
    assert r0['updates'] == r1['updates'] == 3
    for k, v in r0['ema'].items():
        assert torch.equal(v, r1['ema'][k]), 'ranks disagree on ' + k
