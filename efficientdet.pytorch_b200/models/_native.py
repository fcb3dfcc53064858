"""ctypes binding of ``csrc/libeffdet_b200.so`` (the C ABI declared in ``include/effdet_b200.h``).

There is deliberately no fallback: if the shared object is missing, or a tensor is not a CUDA
fp32 tensor, the call raises.  PyTorch only supplies device memory, the current stream and the
device index; every arithmetic kernel on the hot path lives in the shared object.
"""
import ctypes
import os
import subprocess
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.normpath(os.path.join(_HERE, '..', 'csrc'))
SO_PATH = os.path.join(CSRC, 'libeffdet_b200.so')
SOURCES = ['api.cu', 'conv_api.cu', 'conv_simt.cu', 'conv_tc.cu', 'conv_planes.cu', 'pw_gemm.cu', 'pw_wgrad.cu', 'stem.cu', 'dw_fused.cu', 'mbconv_ops.cu', 'se_ops.cu', 'bifpn.cu', 'pipeline.cu',
           'loss.cu', 'detect.cu', 'soft_nms.cu', 'layout.cu', 'optim.cu', 'voc_eval.cu', 'coco_eval.cu']
NVCC_FLAGS = ['-std=c++17', '-O3', '-lineinfo', '-gencode', 'arch=compute_90a,code=sm_90a',
              '-Xcompiler', '-fPIC', '-shared']

ACT_NONE, ACT_RELU, ACT_SWISH, ACT_SIGMOID = 0, 1, 2, 3
FUSE_UP, FUSE_POOL = 0, 1


class EffdetNativeError(RuntimeError):
    pass


def build(force=False, verbose=False):
    """Compile the sm_90a shared object in-tree with nvcc (cross-compiles without a GPU): one object per .cu,
    compiled in parallel and only when stale, then one link step."""
    from concurrent.futures import ThreadPoolExecutor
    import hashlib
    hdrs = [os.path.join(CSRC, 'common.cuh'), os.path.join(CSRC, 'tc_ptx.cuh'), os.path.join(CSRC, 'bitonic.cuh'),
            os.path.join(CSRC, 'block_scan.cuh'),
            os.path.normpath(os.path.join(CSRC, '..', '..', 'include', 'effdet_b200.h'))]
    hdr_blob = b''.join(open(h, 'rb').read() for h in hdrs if os.path.exists(h))
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    flags = [f for f in NVCC_FLAGS if f != '-shared']
    jobs, stamps = [], []
    for s in SOURCES:                      # staleness by CONTENT (file times do not survive the trip to the GPU box)
        src, obj = os.path.join(CSRC, s), os.path.join(CSRC, s[:-3] + '.o')
        digest = hashlib.sha1(open(src, 'rb').read() + hdr_blob + ' '.join(flags).encode()).hexdigest()
        stamp = obj + '.sha1'
        have = open(stamp).read().strip() if os.path.exists(stamp) else ''
        if force or not os.path.exists(obj) or have != digest:
            jobs.append([nvcc] + flags + ['-c', src, '-o', obj])
            stamps.append((stamp, digest))

    def run(cmd):
        if verbose:
            print(' '.join(cmd))
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise EffdetNativeError('nvcc failed:\n' + r.stdout + r.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(run, jobs))
        for stamp, digest in stamps:
            open(stamp, 'w').write(digest)
    objs = [os.path.join(CSRC, s[:-3] + '.o') for s in SOURCES]
    if jobs or not os.path.exists(SO_PATH):
        run([nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', SO_PATH] + objs)
    return SO_PATH


_P = ctypes.c_void_p
_I32 = ctypes.c_int32
_I64 = ctypes.c_int64
_F = ctypes.c_float


class ConvArgs(ctypes.Structure):
    _fields_ = [('x', _P), ('x_bstride', _I64), ('w', _P), ('y', _P), ('y_bstride', _I64), ('z', _P),
                ('bias', _P), ('scale', _P), ('shift', _P), ('a_scale', _P), ('row_scale', _P),
                ('residual', _P), ('r_bstride', _I64), ('mask_src', _P), ('m_bstride', _I64),
                ('B', _I32), ('H', _I32), ('W', _I32), ('Cin', _I32), ('Cout', _I32), ('ksize', _I32), ('act', _I32),
                ('w_tc', _P), ('in_scale', _P), ('in_shift', _P), ('x_planes', _P), ('tc_single', _I32)]


class WgradArgs(ctypes.Structure):
    _fields_ = [('x', _P), ('x_bstride', _I64), ('dy', _P), ('dy_bstride', _I64), ('dw', _P), ('dbias', _P),
                ('a_scale', _P), ('B', _I32), ('H', _I32), ('W', _I32), ('Cin', _I32), ('Cout', _I32), ('ksize', _I32),
                ('precision', _I32), ('ws_x', _P), ('ws_dy', _P), ('in_scale', _P), ('in_shift', _P), ('dy_planes', _P),
                ('x_planes', _P), ('tc_single', _I32), ('ws_dw', _P)]


class BnActBwdArgs(ctypes.Structure):
    _fields_ = [('dy', _P), ('z', _P), ('dz', _P), ('scale', _P), ('shift', _P), ('mean', _P), ('rstd', _P),
                ('dgamma', _P), ('dbeta', _P), ('row_scale', _P), ('gate', _P), ('dmean', _P), ('inv_hw', _F),
                ('B', _I32), ('HW', _I32), ('C', _I32), ('act', _I32)]


class ConvPlanesArgs(ctypes.Structure):
    _fields_ = [('x_planes', _P), ('w_tc', _P), ('bias', _P), ('y', _P), ('y_bstride', _I64), ('y_planes', _P),
                ('mask_planes', _P), ('residual', _P), ('r_bstride', _I64), ('colsum', _P),
                ('B', _I32), ('H', _I32), ('W', _I32), ('Cin', _I32), ('Cout', _I32), ('ksize', _I32), ('act', _I32),
                ('tc_single', _I32), ('y_mask', _P), ('mask_bits', _P)]


class DwFwdArgs(ctypes.Structure):
    _fields_ = [('x', _P), ('in_scale', _P), ('in_shift', _P), ('w_kkc', _P), ('scale', _P), ('shift', _P), ('z', _P),
                ('se_sum', _P), ('B', _I32), ('H', _I32), ('W', _I32), ('C', _I32), ('k', _I32), ('stride', _I32),
                ('pad_t', _I32), ('pad_l', _I32), ('Ho', _I32), ('Wo', _I32), ('se_alpha', _F)]


class DwBwdArgs(ctypes.Structure):
    _fields_ = [('dq', _P), ('z1', _P), ('gate', _P), ('dmean', _P), ('scale1', _P), ('shift1', _P), ('mean1', _P),
                ('rstd1', _P), ('x', _P), ('scale0', _P), ('shift0', _P), ('mean0', _P), ('rstd0', _P), ('w_kkc', _P),
                ('dx', _P), ('dw', _P), ('dgamma1', _P), ('dbeta1', _P), ('dgamma0', _P), ('dbeta0', _P),
                ('inv_hw', _F), ('B', _I32), ('H', _I32), ('W', _I32), ('C', _I32), ('k', _I32), ('stride', _I32),
                ('pad_t', _I32), ('pad_l', _I32), ('Ho', _I32), ('Wo', _I32), ('dx_planes', _P)]


class FuseArgs(ctypes.Structure):
    _fields_ = [('a', _P), ('b', _P), ('c', _P), ('w', _P), ('w_stride', _I32), ('eps', _F), ('out', _P),
                ('B', _I32), ('H', _I32), ('W', _I32), ('C', _I32), ('mode', _I32), ('out_planes', _P)]


class FuseBwdArgs(ctypes.Structure):
    _fields_ = [('dout', _P), ('a', _P), ('b', _P), ('c', _P), ('w', _P), ('w_stride', _I32), ('eps', _F),
                ('da', _P), ('db', _P), ('dc', _P), ('acc_a', _I32), ('acc_b', _I32), ('acc_c', _I32),
                ('dw', _P), ('scratch', _P), ('B', _I32), ('H', _I32), ('W', _I32), ('C', _I32), ('mode', _I32)]


_INT = ctypes.c_int
_TAIL = [_INT, _P]  # (device, stream)

# name -> argument types (everything returns int unless noted); mirrors include/effdet_b200.h
SIGNATURES = {
    'effdet_conv2d': [ctypes.POINTER(ConvArgs)] + _TAIL,
    'effdet_conv2d_multi': [ctypes.POINTER(ConvArgs), _INT] + _TAIL,
    'effdet_conv2d_wgrad': [ctypes.POINTER(WgradArgs)] + _TAIL,
    'effdet_conv_planes_multi': [ctypes.POINTER(ConvPlanesArgs), _INT] + _TAIL,
    'effdet_to_planes': [_P, _I64, _P, _I64, _P, _P, _INT, _INT, _INT] + _TAIL,
    'effdet_conv2d_wgrad_multi': [ctypes.POINTER(WgradArgs), _INT] + _TAIL,
    'effdet_pack_conv_weight': [_P, _P, _P, _INT, _INT, _INT] + _TAIL,
    'effdet_pack_conv_weight_tc': [_P, _P, _P, _INT, _INT, _INT] + _TAIL,
    'effdet_stem_fwd': [_P, _P, _P, _P, _P, _P, _INT, _INT, _INT, _INT] + _TAIL,
    'effdet_stem_wgrad': [_P, _P, _P, _INT, _INT, _INT, _INT] + _TAIL,
    'effdet_pack_dw_weight': [_P, _P, _INT, _INT] + _TAIL,
    'effdet_dwconv_fwd_fused': [ctypes.POINTER(DwFwdArgs)] + _TAIL,
    'effdet_dwconv_bwd_fused': [ctypes.POINTER(DwBwdArgs)] + _TAIL,
    'effdet_bnact_bwd': [ctypes.POINTER(BnActBwdArgs)] + _TAIL,
    'effdet_bn_fold': [_P, _P, _P, _P, _F, _P, _P, _P, _INT] + _TAIL,
    'effdet_add': [_P, _P, _P, _I64] + _TAIL,
    'effdet_relu_bwd': [_P, _P, _P, _I64] + _TAIL,
    'effdet_spatial_reduce_act': [_P, _P, _P, _P, _P, _F, _INT, _INT, _INT] + _TAIL,
    'effdet_se_gate_fwd': [_P] * 7 + [_INT] * 3 + _TAIL,
    'effdet_se_gate_bwd': [_P] * 12 + [_INT] * 3 + _TAIL,
    'effdet_bifpn_fuse_fwd': [ctypes.POINTER(FuseArgs)] + _TAIL,
    'effdet_bifpn_fuse_bwd': [ctypes.POINTER(FuseBwdArgs)] + _TAIL,
    'effdet_focal_loss_fwd': [_P] * 7 + [_INT] * 4 + [_F, _F] + _TAIL,
    'effdet_focal_loss_bwd': [_P] * 9 + [_INT] * 4 + [_F, _F] + _TAIL,
    'effdet_focal_loss_counted_fwd': [_P] * 8 + [_INT] * 4 + [_F, _F] + _TAIL,
    'effdet_focal_loss_counted_bwd': [_P] * 10 + [_INT] * 4 + [_F, _F] + _TAIL,
    'effdet_pack_annots': [_P, _INT, _INT, _P, _P, _INT, _INT] + _TAIL,
    'effdet_sigmoid_bwd': [_P, _P, _P, _I64] + _TAIL,
    'effdet_detect_candidates_batch': [_P] * 8 + [_INT, _INT, _INT, _INT, _F, _F, _F] + _TAIL,
    'effdet_nms_batch': [_P, _P, _P, _INT, _INT, _INT, _INT, ctypes.c_double, _P, _P, _P] + _TAIL,
    'effdet_nms_batch_chunked': [_P, _P, _P] + [_INT] * 5 + [ctypes.c_double, _P, _I64, _P, _P] + _TAIL,
    'effdet_gather_detections_batch': [_P, _P, _P, _P, _P, _INT, _INT, _INT, _P, _P, _P] + _TAIL,
    'effdet_soft_nms_batch': [_P] * 5 + [_INT] * 5 + [ctypes.c_double] * 2 + [_F, _P, _I64] + [_P] * 4 + _TAIL,
    'effdet_soft_nms_batch_classes': [_P] * 5 + [_INT] * 5 + [ctypes.c_double] * 2 + [_F, _P, _I64] + [_P] * 4 + _TAIL,
    'effdet_nms_batch_chunked_classes': [_P] * 4 + [_INT] * 5 + [ctypes.c_double, _P, _I64, _P, _P] + _TAIL,
    'effdet_detect_topk_batch': [_P] * 3 + [_INT] * 3 + [_F] * 3 + [_INT, _INT, _P, _I64] + [_P] * 5 + _TAIL,
    'effdet_multi_sumsq': [_P, _P, _P, _P, _INT, _INT, _P] + _TAIL,
    'effdet_multi_clip_adamw': [_P] * 7 + [_INT, _INT, _P] + [_F] * 8 + [_INT] + _TAIL,
    'effdet_multi_accumulate': [_P] * 5 + [_INT, _INT] + [_P] * 3 + _TAIL,
    'effdet_multi_clip_adamw_dev': [_P] * 7 + [_INT, _INT, _P, _F] + [_P] * 4 + [ctypes.c_double] * 2 + [_F] * 2 + _TAIL,
    'effdet_normalize_pad': [_P, _P, _P, _P, _P, _INT, _INT, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double)] + _TAIL,
    'effdet_resize_normalize_pad': [_P] * 6 + [_INT] * 3 + [ctypes.POINTER(ctypes.c_double)] * 2 + _TAIL,
    'effdet_collate_annots': [_P, _P, _P, _P, _P, _P, _INT, _INT] + _TAIL,
    'effdet_collate_pack_annots': [_P] * 8 + [_INT, _INT] + _TAIL,
    'effdet_frame_transform': [_P] * 4 + [_INT] * 3 + [ctypes.POINTER(ctypes.c_float)] * 2 + _TAIL,
    'effdet_frame_boxes': [_P] * 5 + [_INT] * 4 + [_P, _P] + _TAIL,
    'effdet_eval_select': [_P, _P, _P, _INT, _F, _F, _INT, _INT, _P, _P, _P, _P] + _TAIL,
    'effdet_eval_select_batch': [_P] * 5 + [_INT, _INT, _F, _INT, _INT] + [_P] * 4 + _TAIL,
    'effdet_voc_match': [_P] * 4 + [_INT] * 4 + [ctypes.c_double, _P, _P] + _TAIL,
    'effdet_voc_ap': [_P] * 4 + [_INT, _INT] + [_P] * 3 + [_I64] + _TAIL,
    'effdet_coco_select_batch': [_P] * 6 + [_INT, _INT, ctypes.c_double, _P] + [_INT] * 4 + [_P] * 9 + _TAIL,
    'effdet_coco_match': [_P] * 5 + [_INT, _P, _P] + [_INT] * 3 + [_P, _INT, _INT, _P, _P] + _TAIL,
    'effdet_coco_accumulate': [_P] * 8 + [_INT] * 4 + [_INT] * 3 + [_P] * 3 + [_I64] + _TAIL,
    'effdet_nchw_to_nhwc': [_P, _P, _INT, _INT, _INT, _INT] + _TAIL,
    'effdet_nhwc_to_nchw': [_P, _P, _INT, _INT, _INT, _INT] + _TAIL,
}
PLAIN = {'effdet_version': (ctypes.c_int, []), 'effdet_conv_tc_kpad': (ctypes.c_int, [ctypes.c_int]),
         'effdet_wgrad_tc_geometry_ok': (ctypes.c_int, [ctypes.c_int] * 3), 'effdet_last_error': (ctypes.c_char_p, []),
         'effdet_launch_count': (ctypes.c_uint64, []), 'effdet_reset_launch_count': (None, []),
         'effdet_voc_ap_workspace': (ctypes.c_int64, [ctypes.c_int] * 2),
         'effdet_coco_accumulate_workspace': (ctypes.c_int64, [ctypes.c_int] * 3),
         'effdet_nms_chunked_workspace': (ctypes.c_int64, [ctypes.c_int] * 3),
         'effdet_soft_nms_workspace': (ctypes.c_int64, [ctypes.c_int] * 2),
         'effdet_detect_topk_workspace': (ctypes.c_int64, [ctypes.c_int] * 4)}

_lib = None
_lock = threading.Lock()


def load():
    """Load the shared object (no compute).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(SO_PATH):
                raise EffdetNativeError(
                    'effdet_b200: %s is missing - build it with `python __graft_entry__.py` '
                    '(there is no CPU / PyTorch fallback for the hot path)' % SO_PATH)
            lib = ctypes.CDLL(SO_PATH)
            for name, argtypes in SIGNATURES.items():
                fn = getattr(lib, name)
                fn.argtypes = argtypes
                fn.restype = ctypes.c_int
            for name, (res, argtypes) in PLAIN.items():
                fn = getattr(lib, name)
                fn.argtypes = argtypes
                fn.restype = res
            _lib = lib
    return _lib


def last_error():
    return load().effdet_last_error().decode('utf-8', 'replace')


def launch_count():
    return int(load().effdet_launch_count())


def reset_launch_count():
    load().effdet_reset_launch_count()


def ptr(t):
    """Device pointer of a CUDA fp32 (or explicitly typed) tensor; None passes NULL."""
    if t is None:
        return None
    if not t.is_cuda:
        raise EffdetNativeError('effdet_b200 kernels need CUDA tensors (got %s); there is no CPU path' % t.device)
    return t.data_ptr()


def f32(t, name='tensor'):
    if t is None:
        return None
    if not t.is_cuda or t.dtype != torch.float32:
        raise EffdetNativeError('%s must be a CUDA float32 tensor (got %s on %s)' % (name, t.dtype, t.device))
    if not t.is_contiguous():
        raise EffdetNativeError('%s must be contiguous (shape %s strides %s)' % (name, tuple(t.shape), t.stride()))
    return t.data_ptr()


PROFILER = None   # set to a Profiler() to time every entry point with CUDA events (bench.py)


class Profiler:
    """CUDA-event timing of every C-ABI call on the launching stream (used by bench.py only)."""

    def __init__(self):
        self.recs = []
        self.work = []

    def add(self, name, tag, e0, e1, nbytes=0, flops=0):
        self.recs.append((name, tag, e0, e1))
        self.work.append((nbytes, flops))

    def rooflines(self, hbm_gbs, tensor_tflops):
        """per entry-point class: device ms, algorithmic GB/s and TFLOP/s and the fraction of the measured peaks"""
        out = {}
        for (n, t, e0, e1), (nb, fl) in zip(self.recs, self.work):
            key = n.replace('effdet_', '')
            if t is not None:
                key += ' k%d %d->%d' % (t[5], t[3], t[4])
            v = out.setdefault(key, [0.0, 0, 0.0, 0.0])
            v[0] += e0.elapsed_time(e1)
            v[1] += 1
            v[2] += nb
            v[3] += fl
        res = {}
        for k, (ms, cnt, nb, fl) in out.items():
            if ms <= 0:
                continue
            gbs, tfs = nb / ms / 1e6, fl / ms / 1e9
            res[k] = dict(ms=round(ms, 4), launches=cnt, gb_per_s=round(gbs, 1), hbm_frac=round(gbs / hbm_gbs, 3),
                          tflops=round(tfs, 2), tensor_frac=round(tfs / tensor_tflops, 4))
        return res

    def _ms(self):
        return [(n, t, e0.elapsed_time(e1)) for (n, t, e0, e1) in self.recs]

    def table(self):
        out = {}
        for n, t, ms in self._ms():
            key = n.replace('effdet_', '')
            if t is not None:
                key += ' k%d %d->%d' % (t[5], t[3], t[4])
            v = out.setdefault(key, [0.0, 0])
            v[0] += ms
            v[1] += 1
        return out

    def conv_flops(self, pred):
        fl, ms_tot, n = 0.0, 0.0, 0
        for name, t, ms in self._ms():
            if name in ('effdet_conv2d', 'effdet_conv2d_multi', 'effdet_conv_planes_multi') and t is not None and pred(t):
                fl += 2.0 * t[0] * t[1] * t[2] * t[5] * t[5] * t[3] * t[4]
                ms_tot += ms
                n += 1
        return fl, ms_tot, n


def call(name, dev_tensor, *args, nbytes=0, flops=0):
    """Invoke an entry point on dev_tensor's device and the current stream of that device.
    nbytes / flops: ALGORITHMIC work of this launch (SURVEY.md 8(d)), only used by the bench profiler."""
    lib = load()
    dev = dev_tensor.device.index
    if dev is None:
        dev = torch.cuda.current_device()
    stream = torch.cuda.current_stream(dev)
    prof = PROFILER
    if prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
    rc = getattr(lib, name)(*args, dev, stream.cuda_stream)
    if prof is not None:
        e1.record(stream)
        tag = None
        if name in ('effdet_conv2d', 'effdet_conv2d_wgrad'):
            a = args[0]
            tag = (a.B, a.H, a.W, a.Cin, a.Cout, a.ksize)
        elif name in ('effdet_conv2d_multi', 'effdet_conv2d_wgrad_multi', 'effdet_conv_planes_multi'):
            arr, nl = args[0], args[1]
            pix = sum(arr[i].B * arr[i].H * arr[i].W for i in range(nl))
            tag = (1, pix, 1, arr[0].Cin, arr[0].Cout, arr[0].ksize)      # B*H*W folded into one factor
        if tag is not None and not flops:
            flops = 2.0 * tag[0] * tag[1] * tag[2] * tag[5] * tag[5] * tag[3] * tag[4]
            if not nbytes:
                nbytes = 4.0 * (tag[0] * tag[1] * tag[2] * (tag[3] + tag[4]) + tag[5] * tag[5] * tag[3] * tag[4])
        prof.add(name, tag, e0, e1, nbytes, flops)
    if rc != 0:
        raise EffdetNativeError('%s failed (%d): %s' % (name, rc, last_error()))
