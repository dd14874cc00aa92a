"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own SparseClusterHead (mmdet3d/models/dense_heads/sparse_cluster_head.py), SparseClusterHeadV2 and FSDSeparateHead
(sparse_cluster_head_v2.py) and BasePointBBoxCoder (core/bbox/coders/base_point_bbox_coder.py), compiled unmodified from their sources
on the CPU through oracle/ref_shim.py, with the reference's own build_mlp (ops/sst/sst_ops.py), box3d_multiclass_nms
(core/post_processing/box3d_nms.py) and xywhr2xyxyr (core/bbox/structures/utils.py).  mmdet 2.14 is absent, so what the heads reach of
it is restated minimally: PseudoSampler / AssignResult and the focal / L1 losses from oracle/anchor3d_ref.py, SmoothL1Loss here,
reduce_mean as the identity (no process group; in float64, so that float64 predictions
give float64 losses rather than losses rounded to the fp32 factor's dtype), multi_apply.  points_in_boxes_gpu comes from oracle/roiaware_oracle.py, nms_gpu from
oracle/iou3d_oracle.py; the box stub is oracle/voteseg_ref.py's, extended with cat / to / bev."""
import copy
import types

import numpy as np
import torch
from torch import nn

from oracle import anchor3d_ref as AR
from oracle import iou3d_oracle as IO
from oracle import voteseg_ref as VR
from oracle.ref_shim import _BaseModule, _passthrough_deco, _Registry, available, load, reference_functions  # noqa: F401

_HEAD = None


class _SmoothL1Loss(nn.Module):
    """mmdet 2.14 SmoothL1Loss, reduction 'mean' with avg_factor"""

    def __init__(self, beta=1.0, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.beta, self.loss_weight = beta, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        diff = torch.abs(pred - target)
        loss = torch.where(diff < self.beta, 0.5 * diff * diff / self.beta, diff - 0.5 * self.beta)
        return self.loss_weight * AR._weight_reduce(loss, weight, avg_factor)


_LOSSES = {"FocalLoss": AR._FocalLoss, "L1Loss": AR._L1Loss, "SmoothL1Loss": _SmoothL1Loss}


class Boxes(VR.Boxes):
    """LiDARInstance3DBoxes as the head uses it: voteseg_ref's stub plus `to`, `cat`, `bev` and a box_dim keyword"""

    def __init__(self, tensor, box_dim=7):
        super().__init__(tensor)

    def __getitem__(self, item):
        return Boxes(self.tensor[item])

    def to(self, device):
        return Boxes(self.tensor.to(device))

    @classmethod
    def cat(cls, boxes_list):
        return cls(torch.cat([b.tensor for b in boxes_list], 0))

    @property
    def bev(self):
        return self.tensor[:, [0, 1, 3, 4, 6]]


def load_cluster_head():
    """namespace(SparseClusterHead, SparseClusterHeadV2, FSDSeparateHead, BasePointBBoxCoder, Boxes) of the reference, built on the CPU"""
    global _HEAD
    if _HEAD is not None:
        return _HEAD
    R = load()
    utils = reference_functions("mmdet3d/core/bbox/structures/utils.py", ["limit_period", "xywhr2xyxyr"], {"np": np})
    nms = reference_functions("mmdet3d/core/post_processing/box3d_nms.py", ["box3d_multiclass_nms"],
                              {"np": np, "nms_gpu": IO.nms_gpu, "nms_normal_gpu": IO.nms_normal_gpu})["box3d_multiclass_nms"]
    coder = reference_functions("mmdet3d/core/bbox/coders/base_point_bbox_coder.py", ["BasePointBBoxCoder"],
                                {"BaseBBoxCoder": object})["BasePointBBoxCoder"]

    def build_loss(cfg):
        c = dict(cfg)
        return _LOSSES[c.pop("type")](**c)

    heads = _Registry()
    g = {"BaseModule": _BaseModule, "force_fp32": _passthrough_deco, "build_loss": build_loss, "build_mlp": R.sst_ops.build_mlp,
         "AssignResult": AR._AssignResult, "PseudoSampler": AR._PseudoSampler, "xywhr2xyxyr": utils["xywhr2xyxyr"],
         "box3d_multiclass_nms": nms, "bbox_overlaps_3d": None, "LiDARInstance3DBoxes": Boxes,
         "build_bbox_coder": lambda cfg: coder(**{k: v for k, v in cfg.items() if k != "type"}), "reduce_mean": lambda t: t.double(),
         "np": np, "nn": nn, "copy": copy, "builder": types.SimpleNamespace(build_head=heads.build)}
    v1 = reference_functions("mmdet3d/models/dense_heads/sparse_cluster_head.py", ["SparseClusterHead"], g)
    v2 = reference_functions("mmdet3d/models/dense_heads/sparse_cluster_head_v2.py", ["FSDSeparateHead", "SparseClusterHeadV2"],
                             dict(g, SparseClusterHead=v1["SparseClusterHead"]))
    heads.d.update(v2)
    _HEAD = types.SimpleNamespace(SparseClusterHead=v1["SparseClusterHead"], SparseClusterHeadV2=v2["SparseClusterHeadV2"],
                                  FSDSeparateHead=v2["FSDSeparateHead"], BasePointBBoxCoder=coder, Boxes=Boxes)
    return _HEAD


def build_cluster_head(cfg, train_cfg=None, test_cfg=None):
    """the reference SparseClusterHeadV2 from a bbox_head config dict (type popped), on the CPU, with ConfigDict-like cfgs"""
    from oracle.cluster_head_oracle import Cfg
    R = load_cluster_head()
    c = dict(cfg)
    c.pop("type", None)
    c["train_cfg"] = Cfg(train_cfg) if train_cfg is not None else None
    c["test_cfg"] = Cfg(test_cfg) if test_cfg is not None else None
    c["separate_head"] = dict(c["separate_head"])
    return R.SparseClusterHeadV2(**c)
