"""Focal loss + smooth-L1 of the reference (``models/losses.py``) as two fused sm_90a kernel passes.

``FocalLoss()(classifications[B,A,K], regressions[B,A,4], anchors[1,A,4], annotations[B,G,5])``
returns ``(cls_loss[1], reg_loss[1])`` exactly like the reference (:152); IoU assignment, the
"no annotation -> zero" branch (:54-58), ignore band 0.4..0.5 (:71-84), alpha/gamma = 0.25/2
(:33-34), box targets with the 0.1/0.2 scaling (:116-136) and smooth-L1 beta 1/9 (:140-146) all run on
the device with no host synchronisation and no per-image Python loop.

Any number of annotation rows per image works.  Up to 256 rows the table is staged in shared memory whole; wider
tables are staged in chunks of 256 rows, keeping each anchor's first maximum across the chunks.  The optional
``counts`` ([1 + B] int32 on the device, as ``_ops.pack_annotations`` writes it) names the real images and each
image's annotation rows without a host read: ``counts[0]`` images take part and the losses are their mean, image b
reads only its first ``counts[1 + b]`` rows, and every image past ``counts[0]`` is padding, with no loss and exactly
zero gradients.  That is how ``GraphedTrainStep(max_annotations=...)`` replays short and ragged batches in one graph.
"""
import torch
import torch.nn as nn

from . import _ops


def calc_iou(a, b):
    """IoU[A,G] helper kept for API parity (reference :6-26); the training path computes IoU inside
    the fused assignment kernel."""
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    iw = torch.clamp(torch.min(a[:, 2:3], b[:, 2]) - torch.max(a[:, 0:1], b[:, 0]), min=0)
    ih = torch.clamp(torch.min(a[:, 3:4], b[:, 3]) - torch.max(a[:, 1:2], b[:, 1]), min=0)
    ua = torch.clamp(((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])).unsqueeze(1) + area - iw * ih, min=1e-8)
    return iw * ih / ua


class FocalLoss(nn.Module):
    alpha = 0.25
    gamma = 2.0

    def forward(self, classifications, regressions, anchors, annotations, counts=None):
        return _ops.FocalLossFn.apply(classifications, regressions, anchors, annotations, self.alpha, self.gamma, counts)
