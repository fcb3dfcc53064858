"""``EfficientDet`` -- the detector wrapper of the reference (``models/efficientdet.py``) as a thin host-side shell
around sm_90a kernels.  Same constructor, attributes, call convention and state-dict schema:

  train :  model([images[B,3,H,W], annotations[B,G,5]]) -> (cls_loss[1], reg_loss[1])   (reference :57-68)
           model([images, annotations, counts[1+B] int32]) -> the same, over the first counts[0] images with counts[1+b]
           annotation rows each (models/losses.py); the rest of the batch is padding
  eval  :  model(image[1,3,H,W]) -> [scores[K], classes[K] int64, boxes[K,4]]            (reference :69-86)

What differs underneath: features stay NHWC end to end, the head writes the level-concatenated
``[B, sum(HWA), K]`` / ``[B, sum(HWA), 4]`` tensors directly (no ``torch.cat``), anchors are cached per input
size, and decode + clip + threshold + NMS run on the device for the whole batch with two read-backs.
"""
import math

import torch
import torch.nn as nn

from . import _ops
from .bifpn import BIFPN
from .efficientnet import EfficientNet
from .losses import FocalLoss
from .module import Anchors, BBoxTransform, ClipBoxes
from .retinahead import RetinaHead

# detector name -> backbone name; d7 re-uses the b6 backbone like the reference table (:10-19)
MODEL_MAP = {'efficientdet-d%d' % i: 'efficientnet-b%d' % min(i, 6) for i in range(8)}
_PYRAMID_LEVELS = 5


def _reference_reinit(model):
    """The reference overwrites EVERY conv in the assembled model (backbone included) with
    N(0, sqrt(2 / (k*k*out_channels))) and resets all BatchNorm affines to (1, 0) (reference :47-53)."""
    for mod in model.modules():
        if isinstance(mod, nn.Conv2d):
            fan = mod.kernel_size[0] * mod.kernel_size[1] * mod.out_channels
            mod.weight.data.normal_(0, math.sqrt(2. / fan))
        elif isinstance(mod, nn.BatchNorm2d):
            mod.weight.data.fill_(1)
            mod.bias.data.zero_()


class EfficientDet(nn.Module):
    def __init__(self, num_classes, network='efficientdet-d0', D_bifpn=3, W_bifpn=88, D_class=3, is_training=True,
                 threshold=0.01, iou_threshold=0.5):
        super().__init__()
        # D_class is accepted and ignored, as in the reference (the head depth is fixed at 4 convs)
        self.is_training = is_training
        self.threshold, self.iou_threshold = threshold, iou_threshold
        # registration order backbone -> neck -> bbox_head fixes the state-dict order
        self.backbone = EfficientNet.from_pretrained(MODEL_MAP[network])
        pyramid_channels = self.backbone.get_list_features()[-_PYRAMID_LEVELS:]
        self.neck = BIFPN(in_channels=pyramid_channels, out_channels=W_bifpn, stack=D_bifpn, num_outs=_PYRAMID_LEVELS)
        self.bbox_head = RetinaHead(num_classes=num_classes, in_channels=W_bifpn)
        self.anchors = Anchors()
        self.regressBoxes = BBoxTransform()
        self.clipBoxes = ClipBoxes()
        _reference_reinit(self)
        self.freeze_bn()
        self.criterion = FocalLoss()

    # -- feature extraction ---------------------------------------------------------------------------------
    def extract_feat_nhwc(self, img):
        stages = self.backbone.extract_features_nhwc(img)
        return self.neck.forward_nhwc(stages[-_PYRAMID_LEVELS:])

    def extract_feat(self, img):
        """backbone + neck, returned as logical-NCHW views (reference :94-100)."""
        return tuple(_ops.to_nchw_view(t) for t in self.extract_feat_nhwc(img))

    def freeze_bn(self):
        """BatchNorm always runs on its running statistics (reference :88-92).  Here that is structural -- BN is
        folded into the conv epilogues -- the call only keeps the holder modules in eval mode for parity."""
        for layer in self.modules():
            if isinstance(layer, nn.BatchNorm2d):
                layer.eval()
        _ops.invalidate_caches()

    def train(self, mode=True):
        """nn.Module.train + a reset of the parameter-derived caches: mode switches are where weight surgery through
        `.data` (which the version-keyed caches cannot see) is finished."""
        _ops.invalidate_caches()
        return super().train(mode)

    # -- the two call conventions -----------------------------------------------------------------------------
    def _raw_predictions(self, images):
        cls, reg = self.bbox_head.forward_concat_nhwc(self.extract_feat_nhwc(images))
        return cls, reg, self.anchors(images)

    def _losses(self, images, annotations, counts=None):
        cls, reg, anchors = self._raw_predictions(images)
        return self.criterion(cls, reg, anchors, annotations, counts)

    def _detections(self, image):
        cls, reg, anchors = self._raw_predictions(image)
        found = _ops.detect_batch(cls[:1], reg[:1], anchors, image.shape[2], image.shape[3], self.threshold,
                                  self.iou_threshold)[0]
        if found[0].numel() == 0:
            print('No boxes to NMS')
            return [torch.zeros(0), torch.zeros(0), torch.zeros(0, 4)]
        return found

    def load_state_dict(self, state_dict, *args, **kwargs):
        """Accepts checkpoints written from a DistributedDataParallel-wrapped model as well: the reference's
        `get_state_dict` (utils/helper.py:25-30) only unwraps DataParallel, so under DDP every key it saves carries
        a `module.` prefix that `train.py:235` / `eval.py:374` then cannot load (SURVEY.md 8(f) rank 4)."""
        if len(state_dict) and all(k.startswith('module.') for k in state_dict):
            state_dict = {k[len('module.'):]: v for k, v in state_dict.items()}
        _ops.invalidate_caches()
        return super().load_state_dict(state_dict, *args, **kwargs)

    @torch.no_grad()
    def detect_batch(self, images):
        """Batched inference (SURVEY.md 8(f) rank 3): one network pass over [B,3,H,W], then decode + threshold +
        NMS of all B images in one set of launches and two host reads.  The reference's forward only post-processes
        image 0 (models/efficientdet.py:73-86), which is why eval.py feeds it one image at a time; entry i here equals
        forward(images[i:i+1]).
        -> list of B triples [scores[K_i], classes[K_i] int64, boxes[K_i,4]] on the device (empty tensors when no
        anchor passes the threshold)."""
        cls, reg, anchors = self._raw_predictions(images)
        return _ops.detect_batch(cls, reg, anchors, images.shape[2], images.shape[3], self.threshold,
                                 self.iou_threshold)

    def forward(self, inputs):
        if self.is_training:
            images, annotations, *counts = inputs
            if len(counts) > 1:
                raise _ops.N.EffdetNativeError('EfficientDet: training inputs are [images, annotations] or '
                                               '[images, annotations, counts], got %d elements' % len(inputs))
            return self._losses(images, annotations, *counts)
        return self._detections(inputs)
