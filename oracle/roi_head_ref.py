"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own FSD second stage on the CPU, compiled unmodified from its sources through oracle/ref_shim.py:
GroupCorrectionHead._assign_and_sample (models/roi_heads/fsd_roi_head.py), the whole FullySparseBboxHead class
(models/roi_heads/bbox_heads/fsd_bbox_head.py, its SIRLayer blocks the reference's own), IoUNegPiecewiseSampler
(core/bbox/samplers/iou_neg_piecewise_sampler.py), DeltaXYZWLHRBBoxCoder (core/bbox/coders/delta_xyzwhlr_bbox_coder.py),
rotation_3d_in_axis and xywhr2xyxyr (core/bbox/structures/utils.py).  mmdet 2.14 is absent, so what the stage reaches of it is restated
here: MaxIoUAssigner.assign / assign_wrt_overlaps, AssignResult, RandomSampler (random_choice keeps the k gallery members with the
smallest keys, ties to the lower proposal index: the native sampler's rule, so both sides draw the same subset), SamplingResult,
CrossEntropyLoss(use_sigmoid) and L1Loss, multi_apply, reduce_mean as the identity.  LiDARInstance3DBoxes is a stub with the
reference's corners and, for BboxOverlaps3D(lidar), overlaps with the float64 BEV overlap of oracle/iou3d_oracle.py (itself pinned to
the reference kernel by tests/test_oracle_iou3d_vs_reference.py); nms_gpu is oracle/iou3d_oracle.py's."""
import types

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from oracle import anchor3d_ref as AR
from oracle import iou3d_oracle as IO
from oracle import roi_head_oracle as RO
from oracle.cluster_head_oracle import Cfg
from oracle.ref_shim import _BaseModule, _passthrough_deco, available, load, reference_functions, reference_methods  # noqa: F401

_NS = None


def _utils():
    return reference_functions("mmdet3d/core/bbox/structures/utils.py", ["rotation_3d_in_axis", "xywhr2xyxyr", "limit_period"],
                               {"np": np})


class Boxes:
    """LiDARInstance3DBoxes as the stage uses it (bottom-centre boxes, box_dim columns)"""

    def __init__(self, tensor, box_dim=7, with_yaw=True, origin=None):
        self.tensor = tensor if isinstance(tensor, torch.Tensor) else torch.as_tensor(tensor)
        self.box_dim = self.tensor.shape[-1] if self.tensor.dim() == 2 else box_dim

    def __len__(self):
        return self.tensor.shape[0]

    @property
    def device(self):
        return self.tensor.device

    def to(self, device):
        return Boxes(self.tensor.to(device))

    def clone(self):
        return Boxes(self.tensor.clone())

    @property
    def bev(self):
        return self.tensor[:, [0, 1, 3, 4, 6]]

    @property
    def corners(self):
        """lidar_box3d.py:54-92"""
        dims = self.tensor[:, 3:6]
        corners_norm = torch.from_numpy(np.stack(np.unravel_index(np.arange(8), [2] * 3), axis=1)).to(device=dims.device,
                                                                                                        dtype=dims.dtype)
        corners_norm = corners_norm[[0, 1, 3, 2, 4, 5, 7, 6]]
        corners_norm = corners_norm - dims.new_tensor([0.5, 0.5, 0])
        corners = dims.view([-1, 1, 3]) * corners_norm.reshape([1, 8, 3])
        corners = _utils()["rotation_3d_in_axis"](corners, self.tensor[:, 6], axis=2)
        corners += self.tensor[:, :3].view(-1, 1, 3)
        return corners


class AssignResult:
    def __init__(self, num_gts, gt_inds, max_overlaps, labels=None):
        self.num_gts, self.gt_inds, self.max_overlaps, self.labels = num_gts, gt_inds, max_overlaps, labels


class MaxIoUAssigner:
    """mmdet 2.14 max_iou_assigner.py with BboxOverlaps3D(coordinate='lidar'), ignore_iof_thr -1, gpu_assign_thr -1"""

    def __init__(self, pos_iou_thr, neg_iou_thr, min_pos_iou=.0, gt_max_assign_all=True, ignore_iof_thr=-1, match_low_quality=True,
                 **kwargs):
        self.pos_iou_thr, self.neg_iou_thr, self.min_pos_iou = pos_iou_thr, neg_iou_thr, min_pos_iou
        self.gt_max_assign_all, self.match_low_quality = gt_max_assign_all, match_low_quality

    def assign(self, bboxes, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None):
        overlaps = RO.iou3d(gt_bboxes, bboxes).to(bboxes.dtype)   # LiDARInstance3DBoxes.overlaps(gt, bboxes), in the boxes' dtype
        return self.assign_wrt_overlaps(overlaps, gt_labels)

    def assign_wrt_overlaps(self, overlaps, gt_labels=None):
        num_gts, num_bboxes = overlaps.size(0), overlaps.size(1)
        assigned_gt_inds = overlaps.new_full((num_bboxes, ), -1, dtype=torch.long)
        if num_gts == 0 or num_bboxes == 0:
            max_overlaps = overlaps.new_zeros((num_bboxes, ))
            if num_gts == 0:
                assigned_gt_inds[:] = 0
            assigned_labels = None if gt_labels is None else overlaps.new_full((num_bboxes, ), -1, dtype=torch.long)
            return AssignResult(num_gts, assigned_gt_inds, max_overlaps, labels=assigned_labels)
        max_overlaps, argmax_overlaps = overlaps.max(dim=0)
        gt_max_overlaps, gt_argmax_overlaps = overlaps.max(dim=1)
        assigned_gt_inds[(max_overlaps >= 0) & (max_overlaps < self.neg_iou_thr)] = 0
        pos_inds = max_overlaps >= self.pos_iou_thr
        assigned_gt_inds[pos_inds] = argmax_overlaps[pos_inds] + 1
        if self.match_low_quality:
            for i in range(num_gts):
                if gt_max_overlaps[i] >= self.min_pos_iou:
                    if self.gt_max_assign_all:
                        assigned_gt_inds[overlaps[i, :] == gt_max_overlaps[i]] = i + 1
                    else:
                        assigned_gt_inds[gt_argmax_overlaps[i]] = i + 1
        assigned_labels = None
        if gt_labels is not None:
            assigned_labels = assigned_gt_inds.new_full((num_bboxes, ), -1)
            pos = torch.nonzero(assigned_gt_inds > 0, as_tuple=False).squeeze()
            if pos.numel() > 0:
                assigned_labels[pos] = gt_labels[assigned_gt_inds[pos] - 1]
        return AssignResult(num_gts, assigned_gt_inds, max_overlaps, labels=assigned_labels)


class RandomSampler:
    """mmdet 2.14 BaseSampler + RandomSampler with the key rule in random_choice.  `key_list`: one key tensor per sample, consumed by
    sample() in order.  The negative pieces hand random_choice positions within neg_inds; _sample_neg records neg_inds to map them."""

    def __init__(self, num, pos_fraction, neg_pos_ub=-1, add_gt_as_proposals=True, **kwargs):
        self.num, self.pos_fraction, self.neg_pos_ub, self.add_gt_as_proposals = num, pos_fraction, neg_pos_ub, add_gt_as_proposals
        self.pos_sampler = self.neg_sampler = self
        self.key_list, self.keys, self._map = [], None, None

    def random_choice(self, gallery, num):
        props = gallery if self._map is None else self._map[gallery]
        order = sorted(range(len(gallery)), key=lambda t: (float(self.keys[props[t]]), int(props[t])))
        return gallery[torch.tensor(order[:num], dtype=torch.long)]


class SamplingResult:
    """mmdet 2.14 sampling_result.py"""

    def __init__(self, pos_inds, neg_inds, bboxes, gt_bboxes, assign_result, gt_flags):
        self.pos_inds, self.neg_inds = pos_inds, neg_inds
        self.pos_bboxes, self.neg_bboxes = bboxes[pos_inds], bboxes[neg_inds]
        self.pos_is_gt = gt_flags[pos_inds]
        self.num_gts = gt_bboxes.shape[0]
        self.pos_assigned_gt_inds = assign_result.gt_inds[pos_inds] - 1
        if gt_bboxes.numel() == 0:
            self.pos_gt_bboxes = torch.empty_like(gt_bboxes).view(-1, 4)
        else:
            if len(gt_bboxes.shape) < 2:
                gt_bboxes = gt_bboxes.view(-1, 4)
            self.pos_gt_bboxes = gt_bboxes[self.pos_assigned_gt_inds, :]
        self.pos_gt_labels = assign_result.labels[pos_inds] if assign_result.labels is not None else None

    @property
    def bboxes(self):
        return torch.cat([self.pos_bboxes, self.neg_bboxes])


class _CrossEntropyLoss(nn.Module):
    """mmdet 2.14 CrossEntropyLoss(use_sigmoid=True): binary_cross_entropy with same-shape labels, reduction 'mean' with avg_factor"""

    def __init__(self, use_sigmoid=True, reduction='mean', loss_weight=1.0, **kwargs):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, cls_score, label, weight=None, avg_factor=None):
        loss = F.binary_cross_entropy_with_logits(cls_score, label.type_as(cls_score), reduction='none')
        return self.loss_weight * AR._weight_reduce(loss, None if weight is None else weight.type_as(cls_score), avg_factor)


def load_roi_head():
    """namespace(FullySparseBboxHead, assign_and_sample, IoUNegPiecewiseSampler, build_head, Boxes) of the reference, on the CPU"""
    global _NS
    if _NS is not None:
        return _NS
    R = load()
    u = _utils()
    coder = reference_functions("mmdet3d/core/bbox/coders/delta_xyzwhlr_bbox_coder.py", ["DeltaXYZWLHRBBoxCoder"],
                                {"BaseBBoxCoder": object})["DeltaXYZWLHRBBoxCoder"]
    sampler = reference_functions("mmdet3d/core/bbox/samplers/iou_neg_piecewise_sampler.py", ["IoUNegPiecewiseSampler"],
                                  {"RandomSampler": RandomSampler, "SamplingResult": SamplingResult})["IoUNegPiecewiseSampler"]

    class KeyedSampler(sampler):
        def sample(self, *a, **k):
            self.keys = self.key_list.pop(0)
            return super().sample(*a, **k)

        def _sample_pos(self, assign_result, num_expected, **kwargs):
            self._map = None
            return super()._sample_pos(assign_result, num_expected, **kwargs)

        def _sample_neg(self, assign_result, num_expected, **kwargs):
            neg = torch.nonzero(assign_result.gt_inds == 0, as_tuple=False)
            self._map = neg.squeeze(1) if neg.numel() else neg.view(-1)
            return super()._sample_neg(assign_result, num_expected, **kwargs)

    def build_voxel_encoder(cfg):
        c = dict(cfg)
        c.pop("type")
        return R.SIRLayer(**c)

    def build_loss(cfg):
        c = dict(cfg)
        t = c.pop("type")
        return {"CrossEntropyLoss": _CrossEntropyLoss, "L1Loss": AR._L1Loss}[t](**c)

    def build_bbox_coder(cfg):
        c = dict(cfg)
        c.pop("type")
        return coder(**c)

    def multi_apply(func, *args, **kwargs):
        from functools import partial
        pfunc = partial(func, **kwargs) if kwargs else func
        return tuple(map(list, zip(*map(pfunc, *args))))

    head_cls = reference_functions("mmdet3d/models/roi_heads/bbox_heads/fsd_bbox_head.py", ["FullySparseBboxHead"], {
        "np": np, "nn": nn, "F": F, "BaseModule": _BaseModule, "force_fp32": _passthrough_deco, "LiDARInstance3DBoxes": Boxes,
        "rotation_3d_in_axis": u["rotation_3d_in_axis"], "xywhr2xyxyr": u["xywhr2xyxyr"], "build_loss": build_loss,
        "scatter_v2": R.sst_ops.scatter_v2, "build_mlp": R.sst_ops.build_mlp, "nms_gpu": IO.nms_gpu, "nms_normal_gpu": IO.nms_normal_gpu,
        "build_bbox_coder": build_bbox_coder, "multi_apply": multi_apply, "reduce_mean": lambda t: t, "HEADS": None,
        "builder": types.SimpleNamespace(build_voxel_encoder=build_voxel_encoder)})["FullySparseBboxHead"]
    assign = reference_methods("mmdet3d/models/roi_heads/fsd_roi_head.py", "GroupCorrectionHead", ["_assign_and_sample"],
                               {"F": F, "LiDARInstance3DBoxes": Boxes, "AssignResult": AssignResult})["_assign_and_sample"]

    def build_head(bbox_head, train_cfg=None, test_cfg=None):
        c = dict(bbox_head)
        c.pop("type", None)
        c.pop("max_num", None)
        h = head_cls(**c)
        h.train_cfg, h.test_cfg = Cfg(train_cfg or {}), Cfg(test_cfg or {})
        return h

    def assign_and_sample(train_cfg, proposal_list, gt_bboxes_3d, gt_labels_3d, keys):
        """GroupCorrectionHead._assign_and_sample of the reference with the keys of every sample"""
        a = train_cfg["assigner"]
        self = types.SimpleNamespace(bbox_assigner=[MaxIoUAssigner(**x) for x in a] if isinstance(a, list) else MaxIoUAssigner(**a))
        s = dict(train_cfg["sampler"])
        s.pop("type")
        self.bbox_sampler = KeyedSampler(**s)
        self.bbox_sampler.key_list = list(keys)
        return assign(self, proposal_list, gt_bboxes_3d, gt_labels_3d)

    _NS = types.SimpleNamespace(FullySparseBboxHead=head_cls, build_head=build_head, assign_and_sample=assign_and_sample, Boxes=Boxes,
                                Cfg=Cfg)
    return _NS
