"""CPU-side checks of the drop-in boundary: the shared object loads and exports every symbol the header
declares, the nn.Module mirror has the reference's state-dict schema, and the product refuses to run
without CUDA tensors (no silent fallback).  No GPU needed, no compute calls."""
import os
import re
import subprocess

import pytest
import torch

import effdet_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def native():
    from models import _native
    _native.build()
    return _native


def test_shared_object_exports_every_declared_symbol(native):
    hdr = open(os.path.join(REPO, 'include', 'effdet_b200.h')).read()
    declared = set(re.findall(r'\b(effdet_[a-z0-9_]+)\s*\(', hdr))
    declared -= {'effdet_stream_t'}
    out = subprocess.run(['nm', '-D', '--defined-only', native.SO_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r' T (effdet_[a-z0-9_]+)', out))
    assert declared, 'header parse failed'
    assert declared <= exported, 'declared but not exported: %s' % sorted(declared - exported)
    bound = set(native.SIGNATURES) | set(native.PLAIN)
    assert declared == bound, 'header vs ctypes binding mismatch: %s' % sorted(declared ^ bound)
    lib = native.load()
    assert lib.effdet_version() >= 100
    assert lib.effdet_conv_tc_kpad(36) == 64 and lib.effdet_conv_tc_kpad(720) == 768


def test_ctypes_struct_layout_matches_header(native, tmp_path):
    """every ctypes.Structure mirrors its C struct: a C program compiled from include/effdet_b200.h with gcc prints
    sizeof and the offset of every field, which must equal what ctypes computes for the Python-side declaration"""
    import ctypes
    import subprocess
    pairs = {'effdet_conv_args': native.ConvArgs, 'effdet_wgrad_args': native.WgradArgs,
             'effdet_bnact_bwd_args': native.BnActBwdArgs, 'effdet_fuse_args': native.FuseArgs,
             'effdet_fuse_bwd_args': native.FuseBwdArgs, 'effdet_dw_fwd_args': native.DwFwdArgs,
             'effdet_dw_bwd_args': native.DwBwdArgs, 'effdet_conv_planes_args': native.ConvPlanesArgs}
    for extra in ('PwGemmArgs',):
        if hasattr(native, extra):
            pairs['effdet_pw_gemm_args'] = getattr(native, extra)
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "effdet_b200.h"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / 'layout.c'
    src.write_text('\n'.join(lines))
    exe = tmp_path / 'layout'
    inc = os.path.join(REPO, 'include')
    subprocess.run(['gcc', '-I', inc, str(src), '-o', str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, cls in pairs.items():
        assert int(out[cname]) == ctypes.sizeof(cls), (cname, out[cname], ctypes.sizeof(cls))
        for fname, _ in cls._fields_:
            assert int(out['%s.%s' % (cname, fname)]) == getattr(cls, fname).offset, (cname, fname)


def test_argument_refusals_and_error_plumbing(native):
    """the boundary's error behaviour (include/effdet_b200.h): arguments are validated BEFORE anything touches the
    device, a failing call returns a negative code and leaves its reason in the thread-local effdet_last_error();
    these calls never reach a kernel launch, so they run without a GPU"""
    import ctypes
    lib = native.load()

    def err():
        return lib.effdet_last_error().decode()

    fake = 1 << 20                                           # aligned non-null "pointer"; never dereferenced
    assert lib.effdet_conv2d(None, 0, None) == -1 and 'null' in err()
    assert lib.effdet_conv2d(ctypes.byref(native.ConvArgs()), 0, None) == -1 and 'null' in err()
    dw = native.DwFwdArgs(x=fake, w_kkc=fake, scale=fake, shift=fake, z=fake, se_sum=fake,
                          B=1, H=8, W=8, C=8, k=4, stride=1, pad_t=1, pad_l=1, Ho=8, Wo=8)
    assert lib.effdet_dwconv_fwd_fused(ctypes.byref(dw), 0, None) == -1 and 'k=4' in err()
    dw.C, dw.k = 6, 3
    assert lib.effdet_dwconv_fwd_fused(ctypes.byref(dw), 0, None) == -1 and 'multiple of 4' in err()
    assert lib.effdet_focal_loss_fwd(fake, fake, fake, fake, fake, fake, fake, 1, 100, 20, 1000, 0.25, 2.0, 0, None) == -1
    assert 'G=1000' in err() and '256' in err()
    assert lib.effdet_stem_fwd(fake, fake, fake, fake, fake, fake, 1, 512, 512, 30, 0, None) == -1 and 'C0=30' in err()
    assert lib.effdet_nms_batch(fake, fake, fake, 1, 100, 128, 0, 0.5, fake, fake, fake, 0, None) == -1 and 'nms' in err()
    assert lib.effdet_multi_sumsq(None, None, None, None, 0, 0, None, 0, None) == -1 and 'multi_sumsq' in err()
    assert lib.effdet_add(fake + 4, fake, fake, 64, 0, None) == -1 and 'alignment' in err()
    assert lib.effdet_add(fake, fake, fake, 62, 0, None) == -1 and 'multiple of 4' in err()
    if not torch.cuda.is_available():
        # valid arguments but no device: a CUDA error code and message, not a crash and not a silent success
        assert lib.effdet_add(fake, fake, fake, 64, 0, None) < 0 and 'cuda' in err().lower()


def test_multi_level_convolutions_check_every_level(native):
    """the multi-level dense-convolution entry points refuse, with the single-level message, whatever the single-level
    call refuses on any level -- also when the levels would otherwise share one tensor-core launch -- and they refuse
    before any device work, so these calls run without a GPU"""
    import ctypes
    lib = native.load()

    def err():
        return lib.effdet_last_error().decode()

    fake = 1 << 20                                           # aligned non-null "pointer"; never dereferenced

    def wg(**kw):                                            # a level the TMA-fed weight-gradient kernel would take
        a = native.WgradArgs(x=fake, x_bstride=8 * 8 * 64, dy=fake, dy_bstride=8 * 8 * 64, dw=fake, B=2, H=8, W=8,
                             Cin=64, Cout=64, ksize=3, precision=1, ws_x=fake, ws_dy=fake)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    def wgrad_multi(*levels):
        return lib.effdet_conv2d_wgrad_multi((native.WgradArgs * len(levels))(*levels), len(levels), 0, None)

    assert wgrad_multi(wg(), wg(x=fake + 4)) == -1 and err() == 'wgrad: pointers must be 16-byte aligned'
    assert wgrad_multi(wg(), wg(x_bstride=8 * 8 * 64 + 2)) == -1 and err().startswith('wgrad: batch strides')
    assert wgrad_multi(wg(ksize=5), wg(ksize=5)) == -1 and err() == 'wgrad: ksize 5 not in {1,3}'
    assert wgrad_multi(wg(), wg(B=0)) == -1 and err() == 'wgrad: empty shape'
    assert lib.effdet_conv2d_wgrad(ctypes.byref(wg(W=0)), 0, None) == -1 and err() == 'wgrad: empty shape'
    assert wgrad_multi(wg(), wg(dw=fake + 4096)) == -1 and 'share dw' in err()
    assert lib.effdet_conv2d_wgrad(None, 0, None) == -1 and err() == 'wgrad: null tensor'

    def conv(**kw):                                          # a level the tensor-core implicit GEMM would take
        a = native.ConvArgs(x=fake, x_bstride=8 * 8 * 64, w=fake, y=fake, y_bstride=8 * 8 * 64, B=2, H=8, W=8, Cin=64,
                            Cout=64, ksize=3, w_tc=fake)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    arr = (native.ConvArgs * 2)(conv(), conv(B=0))
    assert lib.effdet_conv2d_multi(arr, 2, 0, None) == -1 and err() == 'conv2d: empty shape'
    arr = (native.ConvArgs * 2)(conv(), conv(y=fake + 4))
    assert lib.effdet_conv2d_multi(arr, 2, 0, None) == -1 and err() == 'conv2d: pointers must be 16-byte aligned'


@pytest.mark.parametrize('net,W,D', [('efficientdet-d0', 64, 2), ('efficientdet-d3', 160, 5)])
def test_state_dict_schema_matches_reference(net, W, D):
    from models import EfficientDet
    m = EfficientDet(num_classes=20, network=net, D_bifpn=D, W_bifpn=W)
    cfg = O.make_config(net, 20, W, D)
    spec = O.state_dict_spec(cfg)          # pinned to the reference by tests/golden/make_golden.py
    sd = m.state_dict()
    assert list(sd.keys()) == [s[0] for s in spec]
    for name, shape, _ in spec:
        assert tuple(sd[name].shape) == tuple(shape), name
    # constructor side effects of the reference (models/efficientdet.py:47-55)
    assert all(not mod.training for mod in m.modules() if isinstance(mod, torch.nn.BatchNorm2d))
    assert m.is_training is True and m.threshold == 0.01 and m.iou_threshold == 0.5
    assert m.backbone.get_list_features()[-5:] == cfg['stage_out'][-5:]


def test_ddp_prefixed_checkpoint_loads():
    """checkpoints saved from a DDP-wrapped model carry `module.` on every key (utils/helper.py:25-30 only
    unwraps DataParallel); the drop-in model accepts both spellings, and still rejects foreign keys"""
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', 20, 64, 2)
    sd = O.init_state_dict(cfg, seed=5)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64)
    m.load_state_dict({'module.' + k: v for k, v in sd.items()})
    got = m.state_dict()
    assert list(got.keys()) == list(sd.keys())
    assert all(torch.equal(got[k], sd[k]) for k in sd)
    with pytest.raises(RuntimeError):
        m.load_state_dict({'model.' + k: v for k, v in sd.items()})


def test_no_cpu_fallback():
    from models import EfficientDet
    from models._native import EffdetNativeError
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    with pytest.raises(EffdetNativeError):
        m(torch.zeros(1, 3, 128, 128))
    from models.losses import FocalLoss
    with pytest.raises(EffdetNativeError):
        FocalLoss()(torch.zeros(1, 9, 4), torch.zeros(1, 9, 4), torch.zeros(1, 9, 4), torch.zeros(1, 1, 5))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(REPO, 'efficientdet.pytorch_b200')
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                src = open(os.path.join(root, f)).read()
                assert 'effdet_oracle' not in src and 'oracle' not in src.replace('oracle/', ''), os.path.join(root, f)


def test_anchor_table_is_bit_exact_on_host():
    from models.module import _anchor_table, Anchors
    a = Anchors()
    for (h, w) in [(512, 512), (384, 640), (1536, 1536)]:
        tab = _anchor_table(h, w, a.pyramid_levels, a.strides, a.sizes, a.ratios, a.scales)
        assert (tab == O.anchors_for(h, w)).all()


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` prints one JSON line with the contract keys: the reference's own modules when
    baseline/_ref is installed (baseline/install_ref.sh), otherwise the oracle port -- and says which."""
    import json
    import sys
    out = subprocess.run([sys.executable, os.path.join(REPO, 'bench.py'), '--impl', 'reference', '--steps', '1',
                          '--warmup', '0', '--cpu-bs', '1'], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    for key in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
                'vs_baseline', 'dtype', 'data', 'config', 'impl', 'cpu_baseline', 'e2e'):
        assert key in line, key
    assert line['impl'] == 'reference' and line['unit'] == 'img/s' and line['value'] > 0
    have_ref = os.path.exists(os.path.join(REPO, 'baseline', '_ref', 'models', 'efficientdet.py'))
    assert line['cpu_baseline']['kind'] == ('reference' if have_ref else 'port') and line['cpu_baseline']['cores'] >= 1
    assert line['e2e']['h2d_bytes_per_step'] == 0 and line['e2e']['d2h_bytes_per_step'] == 0
