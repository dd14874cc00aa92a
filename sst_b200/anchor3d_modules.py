"""The anchor-based SST configs' neck and head (configs/_base_/models/sst_base.py): SECONDFPN (mmdet3d/models/necks/second_fpn.py) and
Anchor3DHead (mmdet3d/models/dense_heads/anchor3d_head.py, train_mixins.py) on libsstb200, with AlignedAnchor3DRangeGenerator
(core/anchor/anchor_3d_generator.py) and DeltaXYZWLHRBBoxCoder (core/bbox/coders/delta_xyzwhlr_bbox_coder.py).

Anchor3DHead keeps the reference's constructor keywords, forward and state-dict keys.  Its targets and losses run natively
(ops.anchor3d_targets, ops.anchor_focal_loss, ops.anchor_reg_dir_loss) with no host sync and no permuted copy of a head output;
get_bboxes is a torch composition over ops.box3d_multiclass_nms.  SECONDFPN is plain torch / cuDNN."""
import numpy as np
import torch
from torch import nn

from . import ops
from .registry import MODELS

NECKS = MODELS


class AlignedAnchor3DRangeGenerator:
    """anchor_3d_generator.py:226-325 with align_corner=False, one range per size, no custom values, one level.  Anchor
    ((y W + x) S + s) R + r = (x_centers[x], y_centers[y], z[s], sizes[s], rotations[r]); every size must share the x / y range, so the
    anchors are separable.  The axes are built once per feature-map size on the CPU with the reference's own torch arithmetic (fp32
    linspace plus half a step), so they are bit-identical to the reference's CPU anchors, and cached on each device."""

    def __init__(self, ranges, sizes=[[1.6, 3.9, 1.56]], scales=[1], rotations=[0, 1.5707963], custom_values=(), reshape_out=True,
                 size_per_range=True, align_corner=False):
        if align_corner or len(custom_values) or not size_per_range or list(scales) != [1]:
            raise ValueError("AlignedAnchor3DRangeGenerator: only align_corner=False, no custom values, size_per_range and scales=[1] are "
                             f"supported, got align_corner={align_corner}, custom_values={custom_values}, "
                             f"size_per_range={size_per_range}, scales={scales}")
        if len(sizes) != len(ranges):
            if len(ranges) != 1:
                raise ValueError(f"AlignedAnchor3DRangeGenerator: {len(ranges)} ranges for {len(sizes)} sizes")
            ranges = ranges * len(sizes)
        if any([r[0], r[1], r[3], r[4]] != [ranges[0][0], ranges[0][1], ranges[0][3], ranges[0][4]] for r in ranges):
            raise ValueError(f"AlignedAnchor3DRangeGenerator: every size must share the x / y range, got {ranges}")
        self.ranges, self.sizes, self.scales, self.rotations = ranges, sizes, scales, rotations
        self.custom_values, self.reshape_out, self.size_per_range, self.align_corner = custom_values, reshape_out, size_per_range, False
        self._cache = {}

    @property
    def num_base_anchors(self):
        return len(self.rotations) * len(self.sizes)

    @property
    def num_levels(self):
        return 1

    def _host_axes(self, H, W):
        xs, ys, zs, whl = None, None, [], []
        for anchor_range, size in zip(self.ranges, self.sizes):
            r = torch.tensor(anchor_range)
            z = torch.linspace(r[2], r[5], 2)
            y = torch.linspace(r[1], r[4], H + 1)
            x = torch.linspace(r[0], r[3], W + 1)
            z += (z[1] - z[0]) / 2
            y += (y[1] - y[0]) / 2
            x += (x[1] - x[0]) / 2
            xs, ys = x[:W], y[:H]
            zs.append(z[0])
            whl.append(torch.tensor(size).reshape(-1, 3)[0] * 1)
        return xs, ys, torch.stack(zs), torch.stack(whl), torch.tensor(self.rotations)

    def axes(self, featmap_size, device):
        """(x_centers [W], y_centers [H], z [S], sizes [S, 3], rotations [R]), fp32 on `device`, cached per (H, W, device)"""
        H, W = (int(v) for v in featmap_size[-2:])
        key = (H, W, str(torch.device(device)))
        if key not in self._cache:
            self._cache[key] = tuple(t.contiguous().to(device) for t in self._host_axes(H, W))
        return self._cache[key]

    def anchors_at(self, featmap_size, index, device):
        """the [len(index), 7] anchors at flat anchor indices ((y W + x) S + s) R + r"""
        xc, yc, z, whl, rot = self.axes(featmap_size, device)
        W, S, R = xc.numel(), z.numel(), rot.numel()
        r, s, cell = index % R, index // R % S, index // (R * S)
        return torch.cat([xc[cell % W, None], yc[cell // W, None], z[s, None], whl[s], rot[r, None]], 1)

    def grid_anchors(self, featmap_sizes, device='cuda'):
        """the reference's reshape_out=False layout: one [1, H, W, S, R, 7] tensor per level"""
        out = []
        for fs in featmap_sizes:
            H, W = (int(v) for v in fs[-2:])
            a = self.anchors_at((H, W), torch.arange(H * W * self.num_base_anchors, device=device), device)
            a = a.view(1, H, W, len(self.sizes), len(self.rotations), 7)
            out.append(a.reshape(-1, 7) if self.reshape_out else a)
        return out


class DeltaXYZWLHRBBoxCoder:
    """delta_xyzwhlr_bbox_coder.py with code_size 7"""

    def __init__(self, code_size=7):
        if code_size != 7:
            raise ValueError(f"DeltaXYZWLHRBBoxCoder: only code_size 7 is supported, got {code_size}")
        self.code_size = code_size

    @staticmethod
    def encode(src_boxes, dst_boxes):
        xa, ya, za, wa, la, ha, ra = torch.split(src_boxes, 1, dim=-1)
        xg, yg, zg, wg, lg, hg, rg = torch.split(dst_boxes, 1, dim=-1)
        za = za + ha / 2
        zg = zg + hg / 2
        diagonal = torch.sqrt(la**2 + wa**2)
        return torch.cat([(xg - xa) / diagonal, (yg - ya) / diagonal, (zg - za) / ha, torch.log(wg / wa), torch.log(lg / la),
                          torch.log(hg / ha), rg - ra], dim=-1)

    @staticmethod
    def decode(anchors, deltas):
        xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
        xt, yt, zt, wt, lt, ht, rt = torch.split(deltas, 1, dim=-1)
        za = za + ha / 2
        diagonal = torch.sqrt(la**2 + wa**2)
        xg = xt * diagonal + xa
        yg = yt * diagonal + ya
        zg = zt * ha + za
        lg = torch.exp(lt) * la
        wg = torch.exp(wt) * wa
        hg = torch.exp(ht) * ha
        rg = rt + ra
        zg = zg - hg / 2
        return torch.cat([xg, yg, zg, wg, lg, hg, rg], dim=-1)


def limit_period(val, offset=0.5, period=np.pi):
    """core/bbox/structures/utils.py:5-19"""
    return val - torch.floor(val / period + offset) * period


def xywhr2xyxyr(boxes_xywhr):
    """core/bbox/structures/utils.py:85-103"""
    boxes = torch.zeros_like(boxes_xywhr)
    half_w, half_h = boxes_xywhr[:, 2] / 2, boxes_xywhr[:, 3] / 2
    boxes[:, 0] = boxes_xywhr[:, 0] - half_w
    boxes[:, 1] = boxes_xywhr[:, 1] - half_h
    boxes[:, 2] = boxes_xywhr[:, 0] + half_w
    boxes[:, 3] = boxes_xywhr[:, 1] + half_h
    boxes[:, 4] = boxes_xywhr[:, 4]
    return boxes


class _AttrDict(dict):
    """the ConfigDict attribute access box3d_multiclass_nms uses (cfg.nms_thr, cfg.use_rotate_nms, cfg.max_num)"""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


def _norm_2d(norm_cfg, num_features):
    cfg = dict(norm_cfg)
    if cfg.get("type") == "BN":   # mmcv's 'BN' is BatchNorm2d
        cfg.pop("type")
        cfg.pop("requires_grad", None)
        return nn.BatchNorm2d(num_features, **cfg)
    return ops.build_norm_layer(cfg, num_features)[1]


@NECKS.register_module()
class SECONDFPN(nn.Module):
    """second_fpn.py:10-93: per input level a deblock = (ConvTranspose2d with kernel = stride = upsample_stride, or a strided Conv2d for
    strides below 1 or use_conv_for_no_stride), the norm, ReLU; the deblocks' outputs concatenated on channels.  State-dict keys
    deblocks.{i}.0 (conv), deblocks.{i}.1 (norm).  init_weights() is the reference's init_cfg: Kaiming for the transposed convs, 1 for
    the norms' weights."""

    def __init__(self, in_channels=[128, 128, 256], out_channels=[256, 256, 256], upsample_strides=[1, 2, 4],
                 norm_cfg=dict(type='BN', eps=1e-3, momentum=0.01), upsample_cfg=dict(type='deconv', bias=False),
                 conv_cfg=dict(type='Conv2d', bias=False), use_conv_for_no_stride=False, init_cfg=None):
        super().__init__()
        if not len(out_channels) == len(upsample_strides) == len(in_channels):
            raise ValueError("SECONDFPN: in_channels, out_channels and upsample_strides need one entry per level")
        up, conv = dict(upsample_cfg), dict(conv_cfg)
        if up.pop("type", "deconv") != "deconv" or conv.pop("type", "Conv2d") not in ("Conv2d", "Conv"):
            raise ValueError(f"SECONDFPN: only deconv upsampling and Conv2d downsampling are supported, got {upsample_cfg}, {conv_cfg}")
        self.in_channels, self.out_channels, self.fp16_enabled = in_channels, out_channels, False
        deblocks = []
        for i, out_channel in enumerate(out_channels):
            stride = upsample_strides[i]
            if stride > 1 or (stride == 1 and not use_conv_for_no_stride):
                layer = nn.ConvTranspose2d(in_channels[i], out_channel, kernel_size=stride, stride=stride, **up)
            else:
                k = int(np.round(1 / stride).astype(np.int64))
                layer = nn.Conv2d(in_channels[i], out_channel, kernel_size=k, stride=k, **conv)
            deblocks.append(nn.Sequential(layer, _norm_2d(norm_cfg, out_channel), nn.ReLU(inplace=True)))
        self.deblocks = nn.ModuleList(deblocks)

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.ConvTranspose2d):
                nn.init.kaiming_normal_(m.weight, a=0, mode='fan_out', nonlinearity='relu')
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            elif isinstance(m, nn.modules.batchnorm._BatchNorm):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0)

    def forward(self, x):
        assert len(x) == len(self.in_channels)
        ups = [deblock(x[i]) for i, deblock in enumerate(self.deblocks)]
        return [torch.cat(ups, dim=1) if len(ups) > 1 else ups[0]]


def _gt_tensor(boxes):
    """[N, 7] fp32 bottom-centre boxes from a LiDARInstance3DBoxes-like object (`.tensor`) or a raw tensor"""
    t = boxes.tensor if hasattr(boxes, "tensor") else boxes
    if t.dim() != 2 or t.shape[1] != 7:
        raise ValueError(f"Anchor3DHead: GT boxes must be [N, 7] (code_size 7), got {tuple(t.shape)}")
    return t.float()


def _check(cond, what):
    if not cond:
        raise ValueError(f"Anchor3DHead: {what}")


@MODELS.register_module()
class Anchor3DHead(nn.Module):
    """anchor3d_head.py:22-565 for the anchor-based SST configs.  forward(feats) -> ([cls_score], [bbox_pred], [dir_cls_preds]) with
    cls_score [B, S R num_classes, H, W], bbox_pred [B, S R 7, H, W], dir_cls_preds [B, S R 2, H, W].

    Supported (anything else raises ValueError here): AlignedAnchor3DRangeGenerator as above; train_cfg.assigner a list with one
    MaxIoUAssigner per size (BboxOverlapsNearest3D, ignore_iof_thr -1, match_low_quality, either gt_max_assign_all) and pos_weight <= 0;
    assign_per_class either way; DeltaXYZWLHRBBoxCoder(code_size=7); loss_cls FocalLoss(use_sigmoid=True); loss_bbox L1Loss; loss_dir
    CrossEntropyLoss(use_sigmoid=False), all with reduction 'mean'; use_direction_classifier and diff_rad_by_sin.

    loss() returns {'loss_cls': [..], 'loss_bbox': [..], 'loss_dir': [..]} (one level).  GT boxes may be LiDARInstance3DBoxes-like
    objects (`.tensor`) or raw [N, 7] bottom-centre tensors.  get_bboxes returns [(bboxes, scores, labels)] per sample, the boxes wrapped
    in input_meta['box_type_3d'] when the meta has one, else a raw [N, 7] tensor; weighted NMS (wnms / wnms_gpu) raises
    NotImplementedError."""

    def __init__(self, num_classes, in_channels, train_cfg, test_cfg, feat_channels=256, use_direction_classifier=True,
                 anchor_generator=dict(type='Anchor3DRangeGenerator', range=[0, -39.68, -1.78, 69.12, 39.68, -1.78], strides=[2],
                                       sizes=[[1.6, 3.9, 1.56]], rotations=[0, 1.57], custom_values=[], reshape_out=False),
                 assigner_per_size=False, assign_per_class=False, diff_rad_by_sin=True, dir_offset=0, dir_limit_offset=1,
                 bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'), loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0),
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=2.0), loss_dir=dict(type='CrossEntropyLoss', loss_weight=0.2),
                 init_cfg=None):
        super().__init__()
        gen = dict(anchor_generator)
        _check(gen.pop("type", None) == "AlignedAnchor3DRangeGenerator", f"anchor_generator must be AlignedAnchor3DRangeGenerator, got "
               f"{anchor_generator.get('type')}")
        coder = dict(bbox_coder)
        _check(coder.pop("type", None) == "DeltaXYZWLHRBBoxCoder", f"bbox_coder must be DeltaXYZWLHRBBoxCoder, got {bbox_coder}")
        _check(use_direction_classifier and diff_rad_by_sin, "use_direction_classifier and diff_rad_by_sin must be True")
        _check(loss_cls.get("type") == "FocalLoss" and loss_cls.get("use_sigmoid", True) and loss_cls.get("gamma", 2.0) == 2.0 and
               loss_cls.get("alpha", 0.25) == 0.25 and loss_cls.get("reduction", "mean") == "mean" and
               set(loss_cls) <= {"type", "use_sigmoid", "gamma", "alpha", "reduction", "loss_weight"},
               f"loss_cls must be FocalLoss(use_sigmoid=True, gamma=2, alpha=0.25), got {loss_cls}")
        _check(loss_bbox.get("type") == "L1Loss" and loss_bbox.get("reduction", "mean") == "mean" and
               set(loss_bbox) <= {"type", "reduction", "loss_weight"}, f"loss_bbox must be L1Loss, got {loss_bbox}")
        _check(loss_dir.get("type") == "CrossEntropyLoss" and not loss_dir.get("use_sigmoid", False) and
               not loss_dir.get("use_mask", False) and loss_dir.get("class_weight") is None and loss_dir.get("reduction", "mean") == "mean"
               and set(loss_dir) <= {"type", "use_sigmoid", "use_mask", "class_weight", "reduction", "loss_weight"},
               f"loss_dir must be CrossEntropyLoss(use_sigmoid=False), got {loss_dir}")
        _check(int(num_classes) >= 1, f"num_classes must be >= 1, got {num_classes}")
        try:
            self.anchor_generator = AlignedAnchor3DRangeGenerator(**gen)
            self.bbox_coder = DeltaXYZWLHRBBoxCoder(**coder)
        except (ValueError, TypeError) as e:
            raise ValueError(f"Anchor3DHead: {e}") from None
        S = len(self.anchor_generator.sizes)
        _check(S <= 8 and len(self.anchor_generator.rotations) <= 8, "at most 8 anchor sizes and 8 rotations are supported")
        self.assigners = None
        if train_cfg is not None:
            assigners = train_cfg.get("assigner")
            _check(isinstance(assigners, (list, tuple)) and len(assigners) == S,
                   f"train_cfg.assigner must be a list of {S} MaxIoUAssigner dicts, one per anchor size")
            allowed = {"type", "iou_calculator", "pos_iou_thr", "neg_iou_thr", "min_pos_iou", "ignore_iof_thr", "gt_max_assign_all",
                       "match_low_quality", "ignore_wrt_candidates", "gpu_assign_thr"}
            for a in assigners:
                _check(a.get("type") == "MaxIoUAssigner" and set(a) <= allowed, f"unsupported assigner {a}")
                calc = dict(a.get("iou_calculator", dict(type="BboxOverlaps2D")))
                _check(calc.get("type") == "BboxOverlapsNearest3D" and calc.get("coordinate", "lidar") == "lidar",
                       f"the assigner's iou_calculator must be BboxOverlapsNearest3D, got {calc}")
                _check(a.get("ignore_iof_thr", -1) == -1 and a.get("match_low_quality", True) and a.get("gpu_assign_thr", -1) == -1,
                       f"ignore_iof_thr must be -1, match_low_quality True and gpu_assign_thr -1, got {a}")
                _check(all(isinstance(a.get(k), (int, float)) and not isinstance(a.get(k), bool)
                           for k in ("pos_iou_thr", "neg_iou_thr")) and isinstance(a.get("min_pos_iou", 0.0), (int, float)),
                       f"pos_iou_thr / neg_iou_thr / min_pos_iou must be numbers, got {a}")
            _check(train_cfg.get("pos_weight", -1) <= 0, f"pos_weight must be <= 0, got {train_cfg.get('pos_weight')}")
            self.assigners = [dict(pos_iou_thr=float(a["pos_iou_thr"]), neg_iou_thr=float(a["neg_iou_thr"]),
                                   min_pos_iou=float(a.get("min_pos_iou", 0.0)), gt_max_assign_all=bool(a.get("gt_max_assign_all", True)))
                              for a in assigners]
        self.in_channels, self.num_classes, self.feat_channels = in_channels, int(num_classes), feat_channels
        self.diff_rad_by_sin, self.use_direction_classifier = diff_rad_by_sin, use_direction_classifier
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.assigner_per_size, self.assign_per_class = assigner_per_size, assign_per_class
        self.dir_offset, self.dir_limit_offset = dir_offset, dir_limit_offset
        self.fp16_enabled, self.use_sigmoid_cls, self.sampling = False, True, False
        self.loss_cls_weight = float(loss_cls.get("loss_weight", 1.0))
        self.loss_bbox_weight = float(loss_bbox.get("loss_weight", 1.0))
        self.loss_dir_weight = float(loss_dir.get("loss_weight", 1.0))
        self.num_anchors = self.anchor_generator.num_base_anchors
        self.box_code_size = self.bbox_coder.code_size
        self.cls_out_channels = self.num_anchors * self.num_classes
        self.conv_cls = nn.Conv2d(self.feat_channels, self.cls_out_channels, 1)
        self.conv_reg = nn.Conv2d(self.feat_channels, self.num_anchors * self.box_code_size, 1)
        self.conv_dir_cls = nn.Conv2d(self.feat_channels, self.num_anchors * 2, 1)

    def init_weights(self):
        """the reference's init_cfg: Normal(std 0.01) for every Conv2d, conv_cls's bias at prior probability 0.01"""
        for m in (self.conv_cls, self.conv_reg, self.conv_dir_cls):
            nn.init.normal_(m.weight, 0, 0.01)
            nn.init.constant_(m.bias, 0)
        nn.init.constant_(self.conv_cls.bias, float(-np.log((1 - 0.01) / 0.01)))

    def forward_single(self, x):
        return self.conv_cls(x), self.conv_reg(x), self.conv_dir_cls(x)

    def forward(self, feats):
        return tuple(map(list, zip(*[self.forward_single(x) for x in feats])))

    def get_targets(self, featmap_size, gt_bboxes, gt_labels, device):
        """ops.anchor3d_targets for the whole batch: (labels, label_weights, bbox_targets, bbox_weights, dir_targets, dir_weights,
        num_total_pos) in the reference's anchor order"""
        if self.assigners is None:
            raise ValueError("Anchor3DHead: training needs a train_cfg")
        boxes = [_gt_tensor(b).to(device) for b in gt_bboxes]
        labels = [lab.to(device).long() for lab in gt_labels]
        xc, yc, z, whl, rot = self.anchor_generator.axes(featmap_size, device)
        asg = self.assigners
        return ops.anchor3d_targets(xc, yc, z, whl, rot, torch.cat(boxes), torch.cat(labels), [b.shape[0] for b in boxes],
                                    self.num_classes, [a["pos_iou_thr"] for a in asg], [a["neg_iou_thr"] for a in asg],
                                    [a["min_pos_iou"] for a in asg], [a["gt_max_assign_all"] for a in asg], self.assign_per_class,
                                    self.dir_offset)

    def loss(self, cls_scores, bbox_preds, dir_cls_preds, gt_bboxes, gt_labels, input_metas=None, gt_bboxes_ignore=None):
        """{'loss_cls': [focal], 'loss_bbox': [L1], 'loss_dir': [cross-entropy]}, each divided by num_total_pos on the device"""
        if len(cls_scores) != 1:
            raise ValueError(f"Anchor3DHead: one feature level is supported, got {len(cls_scores)}")
        if gt_bboxes_ignore is not None:
            raise ValueError("Anchor3DHead: gt_bboxes_ignore is not supported")
        cls_score, bbox_pred, dir_pred = cls_scores[0], bbox_preds[0], dir_cls_preds[0]
        labels, label_w, bbox_t, bbox_w, dir_t, dir_w, ntp = self.get_targets(cls_score.shape[-2:], gt_bboxes, gt_labels, cls_score.device)
        loss_cls = ops.anchor_focal_loss(cls_score, labels, label_w, ntp, self.num_classes, self.loss_cls_weight)
        loss_bbox, loss_dir = ops.anchor_reg_dir_loss(bbox_pred, dir_pred, labels, bbox_t, bbox_w, dir_t, dir_w, ntp, self.num_classes,
                                                      self.train_cfg.get("code_weight"), self.loss_bbox_weight, self.loss_dir_weight)
        return dict(loss_cls=[loss_cls], loss_bbox=[loss_bbox], loss_dir=[loss_dir])

    def get_bboxes(self, cls_scores, bbox_preds, dir_cls_preds, input_metas, cfg=None, rescale=False):
        cfg = _AttrDict(self.test_cfg if cfg is None else cfg)
        if cfg.get("wnms", False) or cfg.get("wnms_gpu", False):
            raise NotImplementedError("Anchor3DHead.get_bboxes: weighted NMS (wnms / wnms_gpu) is not implemented")
        if len(cls_scores) != 1:
            raise ValueError(f"Anchor3DHead: one feature level is supported, got {len(cls_scores)}")
        return [self.get_bboxes_single(cls_scores[0][i].detach(), bbox_preds[0][i].detach(), dir_cls_preds[0][i].detach(), meta, cfg)
                for i, meta in enumerate(input_metas)]

    def get_bboxes_single(self, cls_score, bbox_pred, dir_cls_pred, input_meta, cfg):
        """anchor3d_head.py:432-551 for one level and use_rotate_nms"""
        fs = cls_score.shape[-2:]
        dir_cls_score = torch.max(dir_cls_pred.permute(1, 2, 0).reshape(-1, 2), dim=-1)[1]
        scores = cls_score.permute(1, 2, 0).reshape(-1, self.num_classes).sigmoid()
        bbox_pred = bbox_pred.permute(1, 2, 0).reshape(-1, self.box_code_size)
        inds = torch.arange(scores.shape[0], device=scores.device)
        nms_pre = cfg.get('nms_pre', -1)
        if nms_pre > 0 and scores.shape[0] > nms_pre:
            _, inds = scores.max(dim=1)[0].topk(nms_pre)
            bbox_pred, scores, dir_cls_score = bbox_pred[inds, :], scores[inds, :], dir_cls_score[inds]
        bboxes = self.bbox_coder.decode(self.anchor_generator.anchors_at(fs, inds, scores.device), bbox_pred)
        bboxes_for_nms = xywhr2xyxyr(bboxes[:, [0, 1, 3, 4, 6]])
        scores = torch.cat([scores, scores.new_zeros(scores.shape[0], 1)], dim=1)
        bboxes, scores, labels, dir_scores = ops.box3d_multiclass_nms(bboxes, bboxes_for_nms, scores, cfg.get('score_thr', 0), cfg.max_num,
                                                                      cfg, dir_cls_score)
        if bboxes.shape[0] > 0:
            dir_rot = limit_period(bboxes[..., 6] - self.dir_offset, self.dir_limit_offset, np.pi)
            bboxes[..., 6] = dir_rot + self.dir_offset + np.pi * dir_scores.to(bboxes.dtype)
        if input_meta is not None and 'box_type_3d' in input_meta:
            bboxes = input_meta['box_type_3d'](bboxes, box_dim=self.box_code_size)
        return bboxes, scores, labels

