"""Shared layers of neck and head, anchors and box coding -- H100-native mirror of the pieces of the
reference's ``models/module.py`` that the detector instantiates: ``ConvModule`` (:405-515),
``Anchors`` (:145-180), ``BBoxTransform`` (:9-49), ``ClipBoxes`` (:52-67) and the init helpers
(:518-559).  The reference's dead code (RegressionModel, ClassificationModel, ConvWS2d, GN/SyncBN
registry, anchors_for_shape) is out of scope (SURVEY.md section 2 row 5).
"""
import warnings

import numpy as np
import torch
import torch.nn as nn

from . import _ops
from ._native import ACT_NONE, ACT_RELU


class ConvModule(nn.Module):
    """conv (+bias) -> [norm] -> [ReLU] block.  Only the configuration the detector uses is
    supported natively: no norm layer, order (conv, norm, act), kernel 1 or 3 with "same" padding,
    stride 1, groups 1.  The ``conv`` child is an ``nn.Conv2d`` parameter holder (state-dict key
    ``<name>.conv.weight/bias`` as in the reference)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 bias='auto', conv_cfg=None, norm_cfg=None, activation='relu', inplace=True,
                 order=('conv', 'norm', 'act')):
        super().__init__()
        assert conv_cfg is None or isinstance(conv_cfg, dict)
        assert norm_cfg is None or isinstance(norm_cfg, dict)
        assert isinstance(order, tuple) and len(order) == 3 and set(order) == {'conv', 'norm', 'act'}
        if norm_cfg is not None or (conv_cfg is not None and conv_cfg.get('type', 'Conv') != 'Conv'):
            raise NotImplementedError('ConvModule: norm layers / non-default conv types are never built by '
                                      'EfficientDet (norm_cfg=None, conv_cfg=None) and have no H100 kernel')
        if activation not in (None, 'relu'):
            raise ValueError('{} is currently not supported.'.format(activation))
        self.conv_cfg, self.norm_cfg, self.activation, self.inplace, self.order = conv_cfg, norm_cfg, activation, inplace, order
        self.with_norm = False
        self.with_activatation = activation is not None
        if bias == 'auto':
            bias = True
        self.with_bias = bias
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                              dilation=dilation, groups=groups, bias=bias)
        k = self.conv.kernel_size
        if not (k[0] == k[1] and k[0] in (1, 3) and self.conv.stride == (1, 1) and self.conv.dilation == (1, 1)
                and self.conv.groups == 1 and self.conv.padding == (k[0] // 2, k[0] // 2)):
            raise NotImplementedError('ConvModule: only k in {1,3}, stride 1, "same" padding, groups 1 have an H100 '
                                      'kernel (got k=%s stride=%s pad=%s)' % (k, self.conv.stride, self.conv.padding))
        self.in_channels, self.out_channels = self.conv.in_channels, self.conv.out_channels
        self.kernel_size, self.stride, self.padding = self.conv.kernel_size, self.conv.stride, self.conv.padding
        self.dilation, self.transposed = self.conv.dilation, self.conv.transposed
        self.output_padding, self.groups = self.conv.output_padding, self.conv.groups
        if self.with_activatation:
            self.activate = nn.ReLU(inplace=inplace)

    def forward_nhwc(self, x, activate=True):
        act = ACT_RELU if (activate and self.with_activatation) else ACT_NONE
        return _ops.ConvBiasActFn.apply(x, self.conv.weight, self.conv.bias, act)

    def forward(self, x, activate=True, norm=True):
        return _ops.to_nchw_view(self.forward_nhwc(_ops.to_nhwc(x, 'ConvModule input'), activate))


def xavier_init(module, gain=1, bias=0, distribution='normal'):
    assert distribution in ['uniform', 'normal']
    (nn.init.xavier_uniform_ if distribution == 'uniform' else nn.init.xavier_normal_)(module.weight, gain=gain)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def normal_init(module, mean=0, std=1, bias=0):
    nn.init.normal_(module.weight, mean, std)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def uniform_init(module, a=0, b=1, bias=0):
    nn.init.uniform_(module.weight, a, b)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def kaiming_init(module, mode='fan_out', nonlinearity='relu', bias=0, distribution='normal'):
    assert distribution in ['uniform', 'normal']
    fn = nn.init.kaiming_uniform_ if distribution == 'uniform' else nn.init.kaiming_normal_
    fn(module.weight, mode=mode, nonlinearity=nonlinearity)
    if hasattr(module, 'bias') and module.bias is not None:
        nn.init.constant_(module.bias, bias)


def bias_init_with_prob(prior_prob):
    return float(-np.log((1 - prior_prob) / prior_prob))


def _anchor_table(height, width, levels, strides, sizes, ratios, scales):
    """float64 NumPy recipe of the reference (generate_anchors + shift, models/module.py:183-214,
    252-273) -- kept on the host in float64 and cast once so the result is bit-identical (H6)."""
    chunks = []
    nr, ns = len(ratios), len(scales)
    for lv, stride, base in zip(levels, strides, sizes):
        fh, fw = (height + 2 ** lv - 1) // (2 ** lv), (width + 2 ** lv - 1) // (2 ** lv)
        cell = np.zeros((nr * ns, 4))
        cell[:, 2:] = base * np.tile(scales, (2, nr)).T
        area = cell[:, 2] * cell[:, 3]
        cell[:, 2] = np.sqrt(area / np.repeat(ratios, ns))
        cell[:, 3] = cell[:, 2] * np.repeat(ratios, ns)
        cell[:, 0::2] -= np.tile(cell[:, 2] * 0.5, (2, 1)).T
        cell[:, 1::2] -= np.tile(cell[:, 3] * 0.5, (2, 1)).T
        gx, gy = np.meshgrid((np.arange(0, fw) + 0.5) * stride, (np.arange(0, fh) + 0.5) * stride)
        offs = np.vstack((gx.ravel(), gy.ravel(), gx.ravel(), gy.ravel())).transpose()
        grid = cell.reshape((1, nr * ns, 4)) + offs.reshape((1, offs.shape[0], 4)).transpose((1, 0, 2))
        chunks.append(grid.reshape((-1, 4)))
    table = np.zeros((0, 4)).astype(np.float32)
    for c in chunks:
        table = np.append(table, c, axis=0)
    return np.expand_dims(table, axis=0).astype(np.float32)


class Anchors(nn.Module):
    """``forward(image)`` -> fp32 ``[1, A, 4]`` on the image's device.  The table depends only on
    (H, W), so it is computed once on the host and cached per (H, W, device) instead of being rebuilt
    and re-uploaded every forward (reference models/module.py:161-180)."""

    def __init__(self, pyramid_levels=None, strides=None, sizes=None, ratios=None, scales=None):
        super().__init__()
        self.pyramid_levels = [3, 4, 5, 6, 7] if pyramid_levels is None else pyramid_levels
        self.strides = [2 ** x for x in self.pyramid_levels] if strides is None else strides
        self.sizes = [2 ** (x + 2) for x in self.pyramid_levels] if sizes is None else sizes
        self.ratios = np.array([0.5, 1, 2]) if ratios is None else ratios
        self.scales = np.array([2 ** 0, 2 ** (1.0 / 3.0), 2 ** (2.0 / 3.0)]) if scales is None else scales
        self._cache = {}

    def forward(self, image):
        h, w = int(image.shape[2]), int(image.shape[3])
        key = (h, w, str(image.device))
        hit = self._cache.get(key)
        if hit is None:
            tab = _anchor_table(h, w, self.pyramid_levels, self.strides, self.sizes, self.ratios, self.scales)
            hit = torch.from_numpy(tab).to(image.device)
            self._cache[key] = hit
        return hit


class BBoxTransform(nn.Module):
    """Box decoding constants (std, mean); the arithmetic is fused with clipping / class-max / threshold
    in ``effdet_detect_candidates_batch`` (reference models/module.py:24-49)."""

    def __init__(self, mean=None, std=None):
        super().__init__()
        self.mean = torch.from_numpy(np.array([0, 0, 0, 0]).astype(np.float32)) if mean is None else mean
        self.std = torch.from_numpy(np.array([0.1, 0.1, 0.2, 0.2]).astype(np.float32)) if std is None else std


class ClipBoxes(nn.Module):
    """Marker module for API parity; clipping is fused into the decode kernel (models/module.py:57-67)."""

    def __init__(self, width=None, height=None):
        super().__init__()
