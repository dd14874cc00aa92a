"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own Anchor3DHead (mmdet3d/models/dense_heads/anchor3d_head.py) and AnchorTrainMixin (train_mixins.py), imported
unmodified for their training and decoding path on the CPU, with the reference's own AlignedAnchor3DRangeGenerator
(core/anchor/anchor_3d_generator.py), DeltaXYZWLHRBBoxCoder (core/bbox/coders/delta_xyzwhlr_bbox_coder.py), BboxOverlapsNearest3D
(core/bbox/iou_calculators/iou3d_calculator.py), box3d_multiclass_nms (core/post_processing/box3d_nms.py), limit_period / xywhr2xyxyr
(core/bbox/structures/utils.py) and LiDARInstance3DBoxes.bev / nearest_bev (core/bbox/structures/lidar_box3d.py).

mmdet 2.14 is absent, so the pieces of it the head reaches are restated here: MaxIoUAssigner (assign_wrt_overlaps with the rules of
oracle/anchor3d_oracle.assign), PseudoSampler, bbox_overlaps, FocalLoss (its py_sigmoid_focal_loss path: the reference builds loss_cls
through mmdet's LOSSES), L1Loss, CrossEntropyLoss, images_to_levels and multi_apply.  nms_gpu comes from oracle/iou3d_oracle.py."""
import importlib
import os
import sys
import types
from functools import partial

import numpy as np
import torch
from torch import nn

from oracle import anchor3d_oracle as AO
from oracle import iou3d_oracle as IO
from oracle.ref_shim import REF_ROOT, _Registry, available, load, reference_functions, reference_methods  # noqa: F401

_HEAD = None


def _multi_apply(func, *args, **kwargs):   # mmdet/core/utils/misc.py
    pfunc = partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def _images_to_levels(target, num_levels):   # mmdet/core/anchor/utils.py
    target = torch.stack(target, 0)
    level_targets = []
    start = 0
    for n in num_levels:
        end = start + n
        level_targets.append(target[:, start:end])
        start = end
    return level_targets


def _weight_reduce(loss, weight, avg_factor):   # mmdet 2.14 weight_reduce_loss, reduction 'mean' with avg_factor
    if weight is not None:
        loss = loss * weight
    return loss.sum() / avg_factor


class _FocalLoss(nn.Module):
    """mmdet 2.14 FocalLoss(use_sigmoid=True) on the CPU: one-hot of the labels without the background column, py_sigmoid_focal_loss"""

    def __init__(self, use_sigmoid=True, gamma=2.0, alpha=0.25, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.gamma, self.alpha, self.loss_weight = gamma, alpha, loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        num_classes = pred.size(1)
        t = torch.nn.functional.one_hot(target, num_classes=num_classes + 1)[:, :num_classes].type_as(pred)
        p = pred.sigmoid()
        pt = (1 - p) * t + p * (1 - t)
        fw = (self.alpha * t + (1 - self.alpha) * (1 - t)) * pt.pow(self.gamma)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(pred, t, reduction='none') * fw
        if weight is not None and weight.shape != loss.shape:
            weight = weight.view(-1, 1)
        return self.loss_weight * _weight_reduce(loss, weight, avg_factor)


class _L1Loss(nn.Module):
    def __init__(self, reduction='mean', loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        return self.loss_weight * _weight_reduce(torch.abs(pred - target), weight, avg_factor)


class _CrossEntropyLoss(nn.Module):
    def __init__(self, use_sigmoid=False, use_mask=False, reduction='mean', class_weight=None, loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, cls_score, label, weight=None, avg_factor=None):
        loss = torch.nn.functional.cross_entropy(cls_score, label, reduction='none')
        return self.loss_weight * _weight_reduce(loss, None if weight is None else weight.float(), avg_factor)


_LOSSES = {"FocalLoss": _FocalLoss, "L1Loss": _L1Loss, "CrossEntropyLoss": _CrossEntropyLoss}


class _AssignResult:
    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels


class _MaxIoUAssigner:
    """mmdet 2.14 MaxIoUAssigner for ignore_iof_thr -1 and gpu_assign_thr -1"""

    def __init__(self, pos_iou_thr, neg_iou_thr, min_pos_iou=.0, gt_max_assign_all=True, ignore_iof_thr=-1, ignore_wrt_candidates=True,
                 match_low_quality=True, gpu_assign_thr=-1, iou_calculator=dict(type='BboxOverlaps2D')):
        assert ignore_iof_thr == -1 and match_low_quality and gpu_assign_thr == -1
        self.pos_iou_thr, self.neg_iou_thr, self.min_pos_iou, self.gt_max_assign_all = pos_iou_thr, neg_iou_thr, min_pos_iou, gt_max_assign_all
        self.iou_calculator = _IOU.build(iou_calculator)

    def assign(self, bboxes, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None):
        overlaps = self.iou_calculator(gt_bboxes, bboxes)
        gi = AO.assign(overlaps, self.pos_iou_thr, self.neg_iou_thr, self.min_pos_iou, self.gt_max_assign_all)
        return _AssignResult(gt_bboxes.shape[0], gi, overlaps.max(dim=0)[0])


class _SamplingResult:
    def __init__(self, pos_inds, neg_inds, bboxes, gt_bboxes, assign_result):
        self.pos_inds, self.neg_inds = pos_inds, neg_inds
        self.pos_bboxes, self.neg_bboxes = bboxes[pos_inds], bboxes[neg_inds]
        self.pos_assigned_gt_inds = assign_result.gt_inds[pos_inds] - 1
        self.pos_gt_bboxes = gt_bboxes[self.pos_assigned_gt_inds, :]


class _PseudoSampler:
    def sample(self, assign_result, bboxes, gt_bboxes, **kwargs):
        pos = torch.nonzero(assign_result.gt_inds > 0, as_tuple=False).squeeze(-1).unique()
        neg = torch.nonzero(assign_result.gt_inds == 0, as_tuple=False).squeeze(-1).unique()
        return _SamplingResult(pos, neg, bboxes, gt_bboxes, assign_result)


_IOU = _Registry()


class Boxes:
    """LiDARInstance3DBoxes as the head uses it: `tensor`, and the reference's own `bev` / `nearest_bev`"""

    def __init__(self, tensor, box_dim=7):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]

    def __getitem__(self, item):
        return Boxes(self.tensor[item])


def load_anchor_head():
    """namespace(Anchor3DHead, Boxes, AlignedAnchor3DRangeGenerator, DeltaXYZWLHRBBoxCoder) of the reference, built on the CPU"""
    global _HEAD
    if _HEAD is not None:
        return _HEAD
    load()
    utils = reference_functions("mmdet3d/core/bbox/structures/utils.py", ["limit_period", "xywhr2xyxyr"], {"np": np})
    meth = reference_methods("mmdet3d/core/bbox/structures/lidar_box3d.py", "LiDARInstance3DBoxes", ["bev", "nearest_bev"],
                             {"np": np, "limit_period": utils["limit_period"]})
    Boxes.bev, Boxes.nearest_bev = property(meth["bev"]), property(meth["nearest_bev"])
    iou = reference_functions("mmdet3d/core/bbox/iou_calculators/iou3d_calculator.py", ["BboxOverlapsNearest3D", "bbox_overlaps_nearest_3d"],
                              {"bbox_overlaps": lambda b1, b2, mode='iou', is_aligned=False: AO.bbox_overlaps(b1, b2),
                               "get_box_type": lambda coordinate: (Boxes, None)})
    _IOU.d["BboxOverlapsNearest3D"] = iou["BboxOverlapsNearest3D"]
    gen = reference_functions("mmdet3d/core/anchor/anchor_3d_generator.py", ["Anchor3DRangeGenerator", "AlignedAnchor3DRangeGenerator"],
                              {"mmcv": types.SimpleNamespace(is_list_of=lambda seq, t: all(isinstance(x, t) for x in seq))})
    coder = reference_functions("mmdet3d/core/bbox/coders/delta_xyzwhlr_bbox_coder.py", ["DeltaXYZWLHRBBoxCoder"], {"BaseBBoxCoder": object})
    nms = reference_functions("mmdet3d/core/post_processing/box3d_nms.py", ["box3d_multiclass_nms"],
                              {"np": np, "nms_gpu": IO.nms_gpu, "nms_normal_gpu": IO.nms_normal_gpu})
    anchor_gens, coders, assigners = _Registry(), _Registry(), _Registry()
    anchor_gens.d.update(gen)
    coders.d.update(coder)
    assigners.d["MaxIoUAssigner"] = _MaxIoUAssigner

    def build_loss(cfg):
        c = dict(cfg)
        return _LOSSES[c.pop("type")](**c)

    saved = {k: sys.modules.get(k) for k in ("mmdet3d.core", "mmdet.core", "mmdet.models", "mmdet3d.models.dense_heads", "mmcv.utils",
                                               "mmdet3d.core.bbox", "mmdet3d.core.bbox.structures", "mmdet.core.bbox",
                                               "mmdet.core.bbox.iou_calculators", "mmdet.core.bbox.iou_calculators.builder")}
    bld = sys.modules["mmdet3d.models.builder"]
    old_build_loss = getattr(bld, "build_loss", None)
    bld.build_loss = build_loss

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m

    mod("mmdet3d.core", PseudoSampler=_PseudoSampler, box3d_multiclass_nms=nms["box3d_multiclass_nms"], limit_period=utils["limit_period"],
        xywhr2xyxyr=utils["xywhr2xyxyr"], box3d_multiclass_wnms=None)
    mod("mmdet.core", build_anchor_generator=anchor_gens.build, build_assigner=assigners.build, build_bbox_coder=coders.build,
        build_sampler=None, multi_apply=_multi_apply, images_to_levels=_images_to_levels)
    mod("mmdet.models", HEADS=_Registry(), NECKS=_Registry(), BACKBONES=_Registry())
    mod("mmdet3d.core.bbox")
    mod("mmdet3d.core.bbox.structures", LiDARInstance3DBoxes=Boxes)
    mod("mmdet.core.bbox")
    mod("mmdet.core.bbox.iou_calculators")
    mod("mmdet.core.bbox.iou_calculators.builder", IOU_CALCULATORS=_IOU)
    mod("mmcv.utils", build_from_cfg=None)
    pkg = types.ModuleType("mmdet3d.models.dense_heads")
    pkg.__path__ = [os.path.join(REF_ROOT, "mmdet3d/models/dense_heads")]
    sys.modules["mmdet3d.models.dense_heads"] = pkg
    try:
        head = importlib.import_module("mmdet3d.models.dense_heads.anchor3d_head")
        neck = importlib.import_module("mmdet3d.models.necks.second_fpn") if _load_second_fpn() else None
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in ("mmdet3d.models.dense_heads.anchor3d_head", "mmdet3d.models.dense_heads.train_mixins", "mmdet3d.models.necks.second_fpn"):
            sys.modules.pop(k, None)
        bld.build_loss = old_build_loss
    _HEAD = types.SimpleNamespace(module=head, Anchor3DHead=head.Anchor3DHead, SECONDFPN=neck.SECONDFPN if neck else None, Boxes=Boxes,
                                  AlignedAnchor3DRangeGenerator=gen["AlignedAnchor3DRangeGenerator"],
                                  DeltaXYZWLHRBBoxCoder=coder["DeltaXYZWLHRBBoxCoder"])
    return _HEAD


def _load_second_fpn():
    """second_fpn.py needs mmcv.cnn's build_upsample_layer: add mmcv's 'deconv' (ConvTranspose2d) to the shim's mmcv.cnn"""
    cnn = sys.modules["mmcv.cnn"]

    def build_upsample_layer(cfg, *args, **kwargs):
        c = dict(cfg)
        assert c.pop("type") == "deconv"
        return nn.ConvTranspose2d(*args, **kwargs, **c)
    cnn.build_upsample_layer = build_upsample_layer
    return True


class _Cfg(dict):
    """mmcv ConfigDict's attribute access"""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError:
            raise AttributeError(k)
        return _Cfg(v) if isinstance(v, dict) else v


def build_anchor_head(geom_or_cfg, train_cfg=None, test_cfg=None):
    """the reference Anchor3DHead from oracle/anchor3d_oracle.geometry() or a head config dict (type popped), on the CPU"""
    R = load_anchor_head()
    if "head" in geom_or_cfg:
        cfg, train_cfg, test_cfg = geom_or_cfg["head"], geom_or_cfg["train_cfg"], geom_or_cfg["test_cfg"]
    else:
        cfg = geom_or_cfg
    c = dict(cfg)
    c.pop("type", None)
    return R.Anchor3DHead(train_cfg=_Cfg(train_cfg) if train_cfg is not None else None,
                          test_cfg=_Cfg(test_cfg) if test_cfg is not None else None, **c)
