"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own VoteSegHead (mmdet3d/models/decode_heads/segmentation_head.py) and its base Base3DDecodeHead (decode_head.py),
compiled unmodified from their sources on the CPU, with the reference's own build_mlp (ops/sst/sst_ops.py).  mmdet 2.14 and mmseg are
absent, so the losses the head builds are restated: mmdet's FocalLoss(use_sigmoid=True) and L1Loss reuse oracle/anchor3d_ref.py's
restatements with reduction 'mean' and no avg_factor (a mean over every element), mmseg's CrossEntropyLoss(use_sigmoid=False) is
F.cross_entropy(weight=class_weight, reduction='none') followed by weight_reduce_loss's mean.  points_in_boxes_gpu comes from
oracle/roiaware_oracle.py; the box stub gives `tensor`, indexing and `gravity_center` as LiDARInstance3DBoxes does."""
import types
from abc import ABCMeta, abstractmethod

import torch
from torch import nn

from oracle import anchor3d_ref as AR
from oracle import roiaware_oracle as RA
from oracle.ref_shim import _BaseModule, _passthrough_deco, available, load, reference_functions  # noqa: F401  (available: the skip)

_HEAD = None


class _FocalLoss(AR._FocalLoss):
    """mmdet 2.14 FocalLoss(use_sigmoid=True), reduction 'mean': without avg_factor the mean over all N C elements"""

    def forward(self, pred, target, weight=None, avg_factor=None):
        return super().forward(pred, target, weight, pred.numel() if avg_factor is None else avg_factor)


class _L1Loss(AR._L1Loss):
    """mmdet 2.14 L1Loss, reduction 'mean': without avg_factor the mean over every element"""

    def forward(self, pred, target, weight=None, avg_factor=None):
        return super().forward(pred, target, weight, pred.numel() if avg_factor is None else avg_factor)


class _SegCrossEntropyLoss(nn.Module):
    """mmseg CrossEntropyLoss(use_sigmoid=False, class_weight, loss_weight), 0.14.1 to 1.0 with avg_non_ignore False: the per-point
    weighted cross-entropy, then its plain mean over the points (not divided by the sum of the weights)"""

    def __init__(self, use_sigmoid=False, use_mask=False, reduction='mean', class_weight=None, loss_weight=1.0, avg_non_ignore=False):
        super().__init__()
        assert not use_sigmoid and not use_mask and reduction == 'mean' and not avg_non_ignore
        self.class_weight, self.loss_weight = class_weight, loss_weight

    def forward(self, cls_score, label, weight=None, avg_factor=None, ignore_index=-100):
        cw = None if self.class_weight is None else cls_score.new_tensor(self.class_weight)
        loss = torch.nn.functional.cross_entropy(cls_score, label, weight=cw, reduction='none', ignore_index=ignore_index)
        return self.loss_weight * loss.mean()


_DET_LOSSES = {"FocalLoss": _FocalLoss, "L1Loss": _L1Loss}
_SEG_LOSSES = {"CrossEntropyLoss": _SegCrossEntropyLoss, "FocalLoss": _FocalLoss}


def _build(table, cfg):
    c = dict(cfg)
    return table[c.pop("type")](**c)


class Boxes:
    """LiDARInstance3DBoxes as get_targets uses it: `tensor` (bottom-centre z), boolean indexing, `gravity_center` (lidar_box3d.py:45-51)
    and `points_in_boxes` (lines 348-360) over the roiaware oracle's points_in_boxes_gpu"""

    def __init__(self, tensor, box_dim=None):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]

    def __getitem__(self, item):
        return Boxes(self.tensor[item])

    @property
    def gravity_center(self):
        b = self.tensor
        return torch.cat([b[:, :2], b[:, 2:3] + b[:, 5:6] * 0.5], 1)

    def points_in_boxes(self, points):
        return RA.points_in_boxes_gpu(points.unsqueeze(0), self.tensor[:, :7].unsqueeze(0).to(points.device)).squeeze(0)


class Cfg(dict):
    """mmcv ConfigDict's attribute access"""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def load_voteseg_head():
    """namespace(VoteSegHead, Base3DDecodeHead, Boxes) of the reference, built on the CPU"""
    global _HEAD
    if _HEAD is not None:
        return _HEAD
    R = load()
    g = {"ABCMeta": ABCMeta, "abstractmethod": abstractmethod, "BaseModule": _BaseModule, "auto_fp16": _passthrough_deco,
         "force_fp32": _passthrough_deco, "normal_init": lambda m, mean=0, std=1, bias=0: (nn.init.normal_(m.weight, mean, std),
                                                                                          nn.init.constant_(m.bias, bias)),
         "build_loss": lambda cfg: _build(_SEG_LOSSES, cfg), "nn": nn}
    base = reference_functions("mmdet3d/models/decode_heads/decode_head.py", ["Base3DDecodeHead"], g)["Base3DDecodeHead"]
    head = reference_functions("mmdet3d/models/decode_heads/segmentation_head.py", ["VoteSegHead"],
                               dict(g, Base3DDecodeHead=base, build_det_loss=lambda cfg: _build(_DET_LOSSES, cfg),
                                    build_mlp=R.sst_ops.build_mlp, checkpoint=torch.utils.checkpoint.checkpoint))["VoteSegHead"]
    _HEAD = types.SimpleNamespace(VoteSegHead=head, Base3DDecodeHead=base, Boxes=Boxes)
    return _HEAD


def build_voteseg_head(cfg, train_cfg=None):
    """the reference VoteSegHead from a segmentation_head config dict (type popped), on the CPU, with train_cfg as a ConfigDict"""
    R = load_voteseg_head()
    c = dict(cfg)
    c.pop("type", None)
    head = R.VoteSegHead(**c)
    head.train_cfg = Cfg(train_cfg or {})
    return head
