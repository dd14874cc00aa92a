"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own FSDV2Head (mmdet3d/models/dense_heads/fsd_v2_head.py), compiled unmodified from its source on the CPU through
oracle/ref_shim.py over the reference's SparseClusterHead, FSDSeparateHead and BasePointBBoxCoder as oracle/cluster_head_ref.py loads
them, with the same restated mmdet pieces.  loss_vel is called without avg_factor, so its L1 / SmoothL1 here also restate mmdet 2.14's
weight_reduce_loss for that case, reduction 'mean': (loss * weight).mean(); with avg_factor they are oracle/anchor3d_ref.py's."""
import copy
import types

import numpy as np
import torch
from torch import nn

from oracle import anchor3d_ref as AR
from oracle import cluster_head_ref as CR
from oracle import iou3d_oracle as IO
from oracle.ref_shim import _BaseModule, _passthrough_deco, _Registry, available, load, reference_functions  # noqa: F401

_HEAD = None


def _reduce(loss, weight, avg_factor):
    """mmdet 2.14 weight_reduce_loss, reduction 'mean': over avg_factor when given, else the mean of the weighted elements"""
    if avg_factor is not None:
        return AR._weight_reduce(loss, weight, avg_factor)
    if weight is not None:
        loss = loss * weight
    return loss.mean()


class _L1Loss(nn.Module):
    def __init__(self, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        return self.loss_weight * _reduce(torch.abs(pred - target), weight, avg_factor)


class _SmoothL1Loss(nn.Module):
    def __init__(self, beta=1.0, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.beta, self.loss_weight = beta, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        diff = torch.abs(pred - target)
        loss = torch.where(diff < self.beta, 0.5 * diff * diff / self.beta, diff - 0.5 * self.beta)
        return self.loss_weight * _reduce(loss, weight, avg_factor)


_LOSSES = {"FocalLoss": AR._FocalLoss, "L1Loss": _L1Loss, "SmoothL1Loss": _SmoothL1Loss}


def load_fsdv2_head():
    """namespace(FSDV2Head, Boxes) of the reference, built on the CPU"""
    global _HEAD
    if _HEAD is not None:
        return _HEAD
    R = load()
    C = CR.load_cluster_head()
    utils = reference_functions("mmdet3d/core/bbox/structures/utils.py", ["limit_period", "xywhr2xyxyr"], {"np": np})
    nms = reference_functions("mmdet3d/core/post_processing/box3d_nms.py", ["box3d_multiclass_nms"],
                              {"np": np, "nms_gpu": IO.nms_gpu, "nms_normal_gpu": IO.nms_normal_gpu})["box3d_multiclass_nms"]

    def build_loss(cfg):
        c = dict(cfg)
        return _LOSSES[c.pop("type")](**c)

    heads = _Registry()
    heads.d.update(FSDSeparateHead=C.FSDSeparateHead)
    g = {"BaseModule": _BaseModule, "force_fp32": _passthrough_deco, "build_loss": build_loss, "build_mlp": R.sst_ops.build_mlp,
         "AssignResult": AR._AssignResult, "PseudoSampler": AR._PseudoSampler, "xywhr2xyxyr": utils["xywhr2xyxyr"],
         "box3d_multiclass_nms": nms, "bbox_overlaps_3d": None, "LiDARInstance3DBoxes": CR.Boxes,
         "build_bbox_coder": lambda cfg: C.BasePointBBoxCoder(**{k: v for k, v in cfg.items() if k != "type"}),
         "reduce_mean": lambda t: t.double(), "np": np, "nn": nn, "copy": copy, "builder": types.SimpleNamespace(build_head=heads.build)}
    v1 = reference_functions("mmdet3d/models/dense_heads/sparse_cluster_head.py", ["SparseClusterHead"], g)
    v2 = reference_functions("mmdet3d/models/dense_heads/fsd_v2_head.py", ["FSDV2Head"], dict(g, SparseClusterHead=v1["SparseClusterHead"]))
    _HEAD = types.SimpleNamespace(FSDV2Head=v2["FSDV2Head"], Boxes=CR.Boxes)
    return _HEAD


def build_fsdv2_head(cfg, train_cfg=None, test_cfg=None):
    """the reference FSDV2Head from a bbox_head config dict (type popped), on the CPU, with ConfigDict-like cfgs"""
    from oracle.cluster_head_oracle import Cfg
    R = load_fsdv2_head()
    c = dict(cfg)
    c.pop("type", None)
    c["train_cfg"] = Cfg(train_cfg) if train_cfg is not None else None
    c["test_cfg"] = Cfg(test_cfg) if test_cfg is not None else None
    c["separate_head"] = dict(c["separate_head"])
    return R.FSDV2Head(**c)
