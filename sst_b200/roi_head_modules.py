"""FSD's second stage: GroupCorrectionHead and FullySparseBboxHead (mmdet3d/models/roi_heads/fsd_roi_head.py,
roi_heads/bbox_heads/fsd_bbox_head.py) on libsstb200.

Assignment and sampling of every sample run in one launch (ops.roi_assign_sample; one host sync, for the sampled row counts), the
targets of every sampled row in one launch (ops.roi_head_targets) and the classification, box and corner losses in one fused launch
sequence (ops.roi_head_loss, no host sync).  The SIR blocks are the package's SIRLayer, the MLPs ops.build_mlp, under the reference's
state-dict keys (bbox_head.block_list.{i}.*, bbox_head.conv_cls.*, bbox_head.conv_reg.*).

Randomness.  The reference's samplers draw subsets with torch.randperm, which no native code can reproduce.  Here the caller draws one
key per proposal with torch.rand (from `generator`, torch's global generator by default), and where the reference calls
random_choice(gallery, k) the k gallery members with the smallest keys are kept, ties to the lower proposal index.  That is a uniform
random subset, as randperm(n)[:k] is, reproducible under torch.manual_seed, and it makes the sampler a pure function of its inputs."""
import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from .anchor3d_modules import xywhr2xyxyr
from .cluster_head_modules import reduce_mean
from .registry import MODELS, build_backbone
from .sir_modules import SIRLayer, group_csr


def _refuse(what, name="FullySparseBboxHead"):
    raise ValueError(f"{name}: {what}")


def rotate_z(xyz, angles):
    """rotation_3d_in_axis(points[:, None], angles, axis=2)[:, 0] (structures/utils.py:21-61): (x cos + y sin, -x sin + y cos, z)"""
    s, c = torch.sin(angles), torch.cos(angles)
    return torch.stack([xyz[:, 0] * c + xyz[:, 1] * s, -xyz[:, 0] * s + xyz[:, 1] * c, xyz[:, 2]], 1)


def delta_decode(anchors, deltas):
    """DeltaXYZWLHRBBoxCoder.decode (delta_xyzwhlr_bbox_coder.py:58-91) with the reference's torch ops"""
    xa, ya, za, wa, la, ha, ra = anchors[:, :7].unbind(1)
    xt, yt, zt, wt, lt, ht, rt = deltas[:, :7].unbind(1)
    za = za + ha / 2
    diagonal = torch.sqrt(la ** 2 + wa ** 2)
    xg, yg, zg = xt * diagonal + xa, yt * diagonal + ya, zt * ha + za
    lg, wg, hg = torch.exp(lt) * la, torch.exp(wt) * wa, torch.exp(ht) * ha
    rg = rt + ra
    zg = zg - hg / 2
    out = [xg, yg, zg, wg, lg, hg, rg]
    if anchors.shape[1] > 7:
        out += [t + a for t, a in zip(deltas[:, 7:].unbind(1), anchors[:, 7:].unbind(1))]
    return torch.stack(out, 1)


class RoiSampling:
    """The sampled RoIs of a batch (what the reference keeps as a list of SamplingResult): per row the sample, the proposal box, the
    max IoU, the assigned GT row (-1 on negatives) and its label; positives first within each sample."""

    def __init__(self, batch_idx, bboxes, iou, gt_rows, gt_labels, gt_bboxes, num_pos, num_rows):
        self.batch_idx, self.bboxes, self.iou, self.gt_rows, self.gt_labels = batch_idx, bboxes, iou, gt_rows, gt_labels
        self.gt_bboxes, self.num_pos, self.num_rows = gt_bboxes, num_pos, num_rows


@MODELS.register_module()
class FullySparseBboxHead(nn.Module):
    """fsd_bbox_head.py:19-892 (without get_bboxes_from_tracklet).  get_targets returns its tensors row-aligned with the RoIs:
    bbox_targets, pos_gt_bboxes and pos_gt_labels are [R, ...] with zeros / -1 on negatives, where the reference's are the
    positives only (`t[reg_mask > 0]` of these).  `max_num`, which the FSDv2 Waymo configs put in bbox_head, is accepted and unused
    (the reference's constructor would raise TypeError on it, so those configs' roi_head could not be built there)."""

    def __init__(self, num_classes, num_blocks, in_channels, feat_channels, rel_mlp_hidden_dims, rel_mlp_in_channels, reg_mlp, cls_mlp,
                 with_rel_mlp=True, with_cluster_center=False, with_distance=False, mode='max', xyz_normalizer=[20, 20, 4], act='gelu',
                 geo_input=True, with_corner_loss=False, bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder'),
                 norm_cfg=dict(type='LN', eps=1e-3, momentum=0.01), corner_loss_weight=1.0,
                 loss_bbox=dict(type='SmoothL1Loss', beta=1.0 / 9.0, loss_weight=2.0),
                 loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True, reduction='none', loss_weight=1.0),
                 dropout=0, cls_dropout=0, reg_dropout=0, unique_once=False, init_cfg=None, max_num=None):
        super().__init__()
        if dict(bbox_coder).get('type') != 'DeltaXYZWLHRBBoxCoder' or dict(bbox_coder).get('code_size', 7) != 7:
            _refuse(f"bbox_coder must be DeltaXYZWLHRBBoxCoder with code size 7, got {bbox_coder}")
        lc, lb = dict(loss_cls), dict(loss_bbox)
        if lc.get('type') != 'CrossEntropyLoss' or not lc.get('use_sigmoid', False) or lc.get('reduction', 'mean') != 'mean' or \
                lc.get('class_weight') is not None or lc.get('use_mask', False):
            _refuse(f"loss_cls must be a sigmoid CrossEntropyLoss with reduction 'mean', got {lc}")
        if lb.get('type') not in ('L1Loss', 'SmoothL1Loss') or lb.get('reduction', 'mean') != 'mean':
            _refuse(f"loss_bbox must be L1Loss or SmoothL1Loss with reduction 'mean', got {lb}")
        self.num_classes = num_classes
        self.with_corner_loss = with_corner_loss
        self.box_code_size = 7
        self.use_sigmoid_cls = True
        self.geo_input = geo_input
        self.corner_loss_weight = corner_loss_weight
        self.num_blocks = num_blocks
        self.unique_once = unique_once
        self.loss_cls_weight = float(lc.get('loss_weight', 1.0))
        self.loss_bbox_cfg = lb
        self.train_cfg = self.test_cfg = None
        self.block_list = nn.ModuleList([
            SIRLayer(in_channels=in_channels[i], feat_channels=feat_channels[i], with_distance=with_distance,
                     with_cluster_center=with_cluster_center, with_rel_mlp=with_rel_mlp, rel_mlp_hidden_dims=rel_mlp_hidden_dims[i],
                     rel_mlp_in_channel=rel_mlp_in_channels[i], with_voxel_center=False, voxel_size=[0.1, 0.1, 0.1],
                     point_cloud_range=[-74.88, -74.88, -2, 74.88, 74.88, 4], norm_cfg=norm_cfg, mode=mode, fusion_layer=None,
                     return_point_feats=i != num_blocks - 1, return_inv=False, rel_dist_scaler=10.0, xyz_normalizer=xyz_normalizer,
                     act=act, dropout=dropout) for i in range(num_blocks)])
        end_channel = sum(sum(c) for c in feat_channels)
        self.conv_cls = ops.build_mlp(end_channel, cls_mlp + [1], norm_cfg, True, act=act, dropout=cls_dropout) if cls_mlp is not None \
            else nn.Linear(end_channel, 1)
        self.conv_reg = ops.build_mlp(end_channel, reg_mlp + [7], norm_cfg, True, act=act, dropout=reg_dropout) if reg_mlp is not None \
            else nn.Linear(end_channel, 7)

    def init_weights(self):
        pass

    def forward(self, pts_xyz, pts_features, pts_info, roi_inds, rois):
        """fsd_bbox_head.py:116-173.  roi_inds may hold the extractor's fake -1 rows: they form a group of their own, dropped with the
        empty RoIs.  The non-empty mask and the alignment of the group features to the RoIs run on the device, with no sync."""
        assert pts_features.size(0) > 0
        pts_features, rois = pts_features.float(), rois.float()
        R = rois.shape[0]
        rois = rois[:, 1:]
        rel_xyz = pts_xyz[:, :3] - rois[:, :3][roi_inds]
        coors = roi_inds.long()[:, None]
        bounds = ([-1], [max(R - 1, 0)])
        kw = {}
        if self.unique_once:
            new_coors, unq_inv = ops.unique_rows(coors, bounds=bounds)
            kw = dict(unq_inv_once=unq_inv, new_coors_once=new_coors, csr_once=group_csr(unq_inv, new_coors.shape[0]))
        out_feats = pts_features
        f_cluster = torch.cat([pts_info['local_xyz'], pts_info['boundary_offset'], pts_info['is_in_margin'][:, None], rel_xyz], dim=-1)
        cluster_feat_list = []
        out_coors = None
        for i, block in enumerate(self.block_list):
            in_feats = torch.cat([pts_xyz, out_feats], 1)
            if self.geo_input:
                in_feats = torch.cat([in_feats, f_cluster / 10], 1)
            if i < self.num_blocks - 1:
                out_feats, out_cluster_feats = block(in_feats, coors, f_cluster, **kw)
            else:
                out_cluster_feats, out_coors = block(in_feats, coors, f_cluster, **kw)
            cluster_feat_list.append(out_cluster_feats)
        final_cluster_feats = torch.cat(cluster_feat_list, dim=1)
        out_coors = out_coors.reshape(-1)
        nonempty_roi_mask = self.get_nonempty_roi_mask(out_coors, R)
        cls_score = self.align_roi_feature_and_rois(self.conv_cls(final_cluster_feats), out_coors, R)
        bbox_pred = self.align_roi_feature_and_rois(self.conv_reg(final_cluster_feats), out_coors, R)
        return cls_score, bbox_pred, nonempty_roi_mask

    @staticmethod
    def _slots(out_coors, num_rois):
        """each group's RoI row, num_rois (a scratch row) for the fake -1 group"""
        return torch.where(out_coors >= 0, out_coors, torch.full_like(out_coors, num_rois))

    def get_nonempty_roi_mask(self, out_coors, num_rois):
        mask = torch.zeros(num_rois + 1, dtype=torch.bool, device=out_coors.device)
        mask[self._slots(out_coors, num_rois)] = True
        return mask[:num_rois]

    def align_roi_feature_and_rois(self, features, out_coors, num_rois):
        """fsd_bbox_head.py:186-204: group features to their RoI rows, zeros for empty RoIs.  Every group's features enter the
        result (the fake group's through the dropped scratch row), so the parameters get a gradient, 0 when every RoI is empty, as the
        reference's `features * 0`."""
        new_feature = features.new_zeros((num_rois + 1, features.size(1)))
        new_feature = new_feature.index_put((self._slots(out_coors, num_rois),), features)
        return new_feature[:num_rois]

    def get_targets(self, sampling_results, rcnn_train_cfg, concat=True):
        """fsd_bbox_head.py:343-388 for every sampled row in one launch (ops.roi_head_targets).  Returns (label, bbox_targets,
        bbox_target_batch_idx, pos_gt_bboxes, pos_gt_labels, reg_mask, label_weights, bbox_weights), row-aligned (see the class)."""
        if not concat:
            _refuse("get_targets with concat=False is not supported")
        s = sampling_results
        pos_thrs, neg_thrs = rcnn_train_cfg['cls_pos_thr'], rcnn_train_cfg['cls_neg_thr']
        if isinstance(pos_thrs, float):
            pos_thrs, neg_thrs = [pos_thrs] * self.num_classes, [neg_thrs] * self.num_classes
        label, reg_mask, bbox_targets, pos_gt = ops.roi_head_targets(s.bboxes, s.iou, s.gt_rows, s.gt_labels, s.gt_bboxes, pos_thrs,
                                                                     neg_thrs)
        R = label.shape[0]
        label_weights = torch.ones_like(label) / max(float(R), 1.0)
        bbox_weights = (reg_mask > 0).float()
        bbox_weights = bbox_weights / torch.clamp(bbox_weights.sum(), min=1.0)
        return (label, bbox_targets, s.batch_idx.int(), pos_gt, s.gt_labels, reg_mask, label_weights, bbox_weights)

    def loss(self, cls_score, bbox_pred, nonempty_roi_mask, rois, labels, bbox_targets, pos_batch_idx, pos_gt_bboxes, pos_gt_labels,
             reg_mask, label_weights, bbox_weights):
        """fsd_bbox_head.py:207-330 in one fused launch sequence, no host sync.  The classification weights are the non-empty mask and
        its average factor the RoI count, the box average factor the device count of positives on non-empty RoIs (each optionally
        reduce_mean'd across ranks); a term without rows is exactly 0 with a zero gradient."""
        cfg = self.train_cfg or {}
        R = cls_score.shape[0]
        assert R > 0
        dev = cls_score.device
        cls_avg = torch.full((1,), float(R), dtype=torch.float32, device=dev)
        if cfg.get('sync_cls_avg_factor', False):
            cls_avg = reduce_mean(cls_avg)
        pos = (reg_mask > 0) & nonempty_roi_mask
        num_pos = pos.sum().float()
        reg_avg = num_pos.reshape(1)
        if cfg.get('sync_reg_avg_factor', False):
            reg_avg = reduce_mean(reg_avg)
        corner_class = -1
        if self.with_corner_loss and cfg.get('corner_loss_only_car', True):
            corner_class = list(cfg['class_names']).index('Car')
        lb = self.loss_bbox_cfg
        lcfg = ops.RoiLossConfig(self.loss_cls_weight, float(lb.get('loss_weight', 1.0)), lb['type'] == 'SmoothL1Loss',
                                 float(lb.get('beta', 1.0)), self.with_corner_loss, corner_class, self.corner_loss_weight,
                                 cfg.get('rcnn_code_weights', None))
        losses = ops.roi_head_loss(cls_score, bbox_pred, nonempty_roi_mask, labels, reg_mask, bbox_targets, pos_gt_bboxes, pos_gt_labels,
                                   rois[:, 1:], cls_avg, reg_avg, lcfg)
        out = dict(loss_rcnn_cls=losses[0], num_pos_rois=num_pos, num_neg_rois=R - num_pos, loss_rcnn_bbox=losses[1])
        if self.with_corner_loss:
            out['loss_rcnn_corner'] = losses[2]
        return out

    def decode_from_rois(self, rois, bbox_pred):
        """fsd_bbox_head.py:871-892: a 9-column RoI keeps its velocity (zero predicted delta)"""
        roi_boxes = rois[:, 1:]
        assert roi_boxes.size(1) in (7, 9)
        local = roi_boxes.clone().detach()
        local[:, 0:3] = 0
        if local.size(1) == 9:
            bbox_pred = F.pad(bbox_pred, (0, 2), 'constant', 0)
        boxes = delta_decode(local, bbox_pred)
        xyz = rotate_z(boxes[:, 0:3], roi_boxes[:, 6] + np.pi / 2) + roi_boxes[:, 0:3]
        return torch.cat([xyz, boxes[:, 3:]], 1)

    def get_bboxes(self, rois, cls_score, bbox_pred, valid_roi_mask, class_labels, class_pred, img_metas, cfg=None):
        """fsd_bbox_head.py:581-684 for a batch of one: every class of multi_class_nms (or the one of single_class_nms) is a segment of
        one ops.nms_bev call; the output keeps the reference's order, class by class, each in keep order."""
        assert rois.size(0) == cls_score.size(0) == bbox_pred.size(0)
        assert isinstance(class_labels, list) and isinstance(class_pred, list) and len(class_labels) == len(class_pred) == 1
        cfg = self.test_cfg if cfg is None else cfg
        cls_score = cls_score.sigmoid()
        if (self.test_cfg or cfg).get('rcnn_score_nms', False):
            class_pred[0] = cls_score.squeeze(1)
        rois, cls_score, bbox_pred = rois[valid_roi_mask], cls_score[valid_roi_mask], bbox_pred[valid_roi_mask]
        labels, probs = class_labels[0][valid_roi_mask], class_pred[0][valid_roi_mask]
        box_type = img_metas[0].get('box_type_3d') if img_metas and img_metas[0] is not None else None
        wrap = (lambda b: box_type(b, b.size(1))) if box_type is not None else (lambda b: b)
        if rois.numel() == 0:
            return [(wrap(rois[:, 1:]), probs, labels)]
        boxes = self.decode_from_rois(rois, bbox_pred)
        score = cls_score.view(-1)
        multi = cfg.get('multi_class_nms', False) or self.num_classes > 1
        sel = self._nms(probs, labels, boxes, cfg['score_thr'], cfg['nms_thr'], cfg['use_rotate_nms'], multi)
        return [(wrap(boxes[sel]), score[sel], labels[sel])]

    def _nms(self, probs, labels, boxes, score_thr, nms_thr, rotated, multi):
        K = self.num_classes if multi else 1
        score_t = list(score_thr) if isinstance(score_thr, (list, tuple)) else [score_thr] * K
        nms_t = list(nms_thr) if isinstance(nms_thr, (list, tuple)) else [nms_thr] * K
        if not multi and not isinstance(score_thr, float):
            _refuse(f"single_class_nms needs a float score_thr, got {score_thr}")
        dev = probs.device
        if multi:
            thr = torch.tensor(score_t, dtype=probs.dtype, device=dev)
            ok = (labels >= 0) & (labels < K)
            keep = ok & (probs >= thr[labels.clamp(0, K - 1)])
            seg = labels
        else:
            keep = probs >= score_t[0]
            seg = torch.zeros_like(labels)
        idx = keep.nonzero(as_tuple=False).view(-1)
        if not multi and nms_t[0] is None:
            return idx
        # per segment by descending score (nms_gpu's sort), then segment by segment
        order = torch.sort(probs[idx], descending=True, stable=True)[1]
        idx = idx[order]
        idx = idx[torch.sort(seg[idx], stable=True)[1]]
        sizes = torch.bincount(seg[idx], minlength=K).tolist() if idx.numel() else [0] * K
        bev = torch.stack([boxes[idx, 0], boxes[idx, 1], boxes[idx, 3], boxes[idx, 4], boxes[idx, 6]], 1)
        off = [0]
        for n in sizes:
            off.append(off[-1] + n)
        kept = ops.nms_bev(xywhr2xyxyr(bev), off, nms_t, rotated=rotated)
        return idx[kept]


@MODELS.register_module()
class GroupCorrectionHead(nn.Module):
    """fsd_roi_head.py:14-296.  train_cfg.assigner: one MaxIoUAssigner (BboxOverlaps3D, lidar) per class, or one over every GT;
    train_cfg.sampler: IoUNegPiecewiseSampler.  _assign_and_sample draws its keys from `generator` (see the module docstring)."""

    def __init__(self, num_classes=3, roi_extractor=None, bbox_head=None, train_cfg=None, test_cfg=None, pretrained=None, init_cfg=None):
        super().__init__()
        self.num_classes = num_classes
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        ext = dict(roi_extractor)
        if ext.pop('with_virtual', False):
            _refuse("roi_extractor with_virtual=True is not supported", "GroupCorrectionHead")
        self.roi_extractor = build_backbone(ext)
        bh = dict(bbox_head)
        if bh.pop('type', 'FullySparseBboxHead') != 'FullySparseBboxHead':
            _refuse(f"bbox_head must be FullySparseBboxHead, got {bbox_head.get('type')}", "GroupCorrectionHead")
        self.bbox_head = FullySparseBboxHead(**bh)
        self.bbox_head.train_cfg, self.bbox_head.test_cfg = train_cfg, test_cfg
        self.sample_cfg = self._sample_cfg(train_cfg) if train_cfg else None

    @property
    def with_bbox(self):
        return True

    def _sample_cfg(self, cfg):
        name = "GroupCorrectionHead"
        assigners = cfg['assigner']
        per_class = isinstance(assigners, (list, tuple))
        assigners = list(assigners) if per_class else [assigners]
        for a in assigners:
            a = dict(a)
            iou = dict(a.get('iou_calculator', {}))
            if a.get('type') != 'MaxIoUAssigner' or iou.get('type') != 'BboxOverlaps3D' or iou.get('coordinate') != 'lidar':
                _refuse(f"assigners must be MaxIoUAssigner over BboxOverlaps3D(lidar), got {a}", name)
            if a.get('ignore_iof_thr', -1) > 0 or not a.get('match_low_quality', True) or not a.get('gt_max_assign_all', True) or \
                    isinstance(a.get('neg_iou_thr'), (list, tuple)) or a.get('gpu_assign_thr', -1) > 0:
                _refuse(f"assigner setting not supported: {a}", name)
        s = dict(cfg['sampler'])
        if s.get('type') != 'IoUNegPiecewiseSampler':
            _refuse(f"sampler must be IoUNegPiecewiseSampler, got {s.get('type')}", name)
        if s.get('add_gt_as_proposals', False):
            _refuse("add_gt_as_proposals=True is not supported", name)
        if s.get('neg_pos_ub', -1) >= 0:
            _refuse(f"neg_pos_ub >= 0 is not supported, got {s.get('neg_pos_ub')}", name)
        if not s.get('return_iou', False):
            _refuse("the sampler must have return_iou=True (get_targets reads the IoU)", name)
        fr, th = list(s['neg_piece_fractions']), list(s['neg_iou_piece_thrs'])
        # With at most 3 pieces, fractions >= 0 and sum(fr[:-1]) <= 1, the reference's carry-over never asks for more than the
        # sample's num rows (the proof is at sstb200_roi_assign_sample); with 4 it can, and the native sampler refuses them.
        if not 1 <= len(fr) <= 3:
            _refuse(f"1 to 3 IoU pieces are supported, got {len(fr)}", name)
        if any(f < 0 for f in fr) or sum(fr[:-1]) > 1 or any(th[i] < th[i + 1] for i in range(len(th) - 1)):
            _refuse(f"neg_piece_fractions must be >= 0 and sum to at most 1 before the last, and neg_iou_piece_thrs descend, got {fr} "
                    f"and {th}", name)
        if cfg.get('class_wise_cls_weights') is not None or cfg.get('class_wise_box_weights') is not None:
            _refuse("class_wise_cls_weights / class_wise_box_weights are not supported", name)
        return ops.RoiSampleConfig([a['pos_iou_thr'] for a in assigners], [a['neg_iou_thr'] for a in assigners],
                                   [a.get('min_pos_iou', 0.0) for a in assigners], per_class, s['num'], s['pos_fraction'], fr, th)

    def forward_train(self, pts_xyz, pts_feats, pts_batch_idx, img_metas, proposal_list, gt_bboxes_3d, gt_labels_3d, generator=None):
        sample_results = self._assign_and_sample(proposal_list, gt_bboxes_3d, gt_labels_3d, generator=generator)
        return self._bbox_forward_train(pts_xyz, pts_feats, pts_batch_idx, sample_results)['loss_bbox']

    def simple_test(self, pts_xyz, pts_feats, pts_batch_inds, img_metas, proposal_list, gt_bboxes_3d, gt_labels_3d, **kwargs):
        assert len(proposal_list) == 1, 'only support bsz==1 to make cls_preds and labels_3d consistent with bbox_results'
        boxes = getattr(proposal_list[0][0], 'tensor', proposal_list[0][0])
        rois = torch.cat([boxes.new_zeros((boxes.shape[0], 1)), boxes], 1)
        cls_preds, labels_3d = [proposal_list[0][1]], [proposal_list[0][2]]
        if len(rois) == 0:
            rois = torch.tensor([[0, 0, 0, 5, 1, 1, 1, 0]], dtype=rois.dtype, device=rois.device)
            cls_preds = [torch.tensor([0.0], dtype=torch.float32, device=rois.device)]
            labels_3d = [torch.tensor([0], dtype=torch.int64, device=rois.device)]
        res = self._bbox_forward(pts_xyz, pts_feats, pts_batch_inds, rois)
        bbox_list = self.bbox_head.get_bboxes(rois, res['cls_score'], res['bbox_pred'], res['valid_roi_mask'], labels_3d, cls_preds,
                                              img_metas, cfg=self.test_cfg)
        return [dict(boxes_3d=b.to('cpu'), scores_3d=s.cpu(), labels_3d=l.cpu()) for b, s, l in bbox_list]  # bbox3d2result

    def _bbox_forward_train(self, pts_xyz, pts_feats, batch_idx, sampling_results):
        s = sampling_results
        rois = torch.cat([s.batch_idx.to(s.bboxes.dtype)[:, None], s.bboxes], 1)
        res = self._bbox_forward(pts_xyz, pts_feats, batch_idx, rois)
        targets = self.bbox_head.get_targets(s, self.train_cfg)
        res.update(loss_bbox=self.bbox_head.loss(res['cls_score'], res['bbox_pred'], res['valid_roi_mask'], rois, *targets))
        return res

    def _bbox_forward(self, pts_xyz, pts_feats, batch_idx, rois):
        assert pts_xyz.size(0) == pts_feats.size(0) == batch_idx.size(0)
        ext_pts_inds, ext_pts_roi_inds, ext_pts_info = self.roi_extractor(pts_xyz[:, :3], batch_idx, rois[:, :8],
                                                                          batch_size=1 if not self.training else None)
        # the extractor's fake rows carry index -1: they gather the last point, as in the reference
        cls_score, bbox_pred, valid_roi_mask = self.bbox_head(pts_xyz[ext_pts_inds], pts_feats[ext_pts_inds], ext_pts_info,
                                                              ext_pts_roi_inds, rois)
        return dict(cls_score=cls_score, bbox_pred=bbox_pred, valid_roi_mask=valid_roi_mask)

    def _assign_and_sample(self, proposal_list, gt_bboxes_3d, gt_labels_3d, generator=None):
        """fsd_roi_head.py:213-296 for the whole batch in one launch.  A sample without proposals gets the fake box
        [0, 0, 5, 1, 1, 1, 0] (+ zero velocity) with label 0.  One host sync."""
        assert len(proposal_list) == len(gt_bboxes_3d)
        boxes, labels = [], []
        for p in proposal_list:
            b = getattr(p[0], 'tensor', p[0])
            assert b.size(1) in (7, 9)
            if len(b) == 0:
                b = torch.tensor([[0, 0, 5, 1, 1, 1, 0, 0, 0][:b.size(1)]], dtype=torch.float32, device=b.device)
                lab = torch.tensor([0], dtype=torch.int64, device=b.device)
            else:
                lab = p[2]
            boxes.append(b.float())
            labels.append(lab.long())
        props, plab = torch.cat(boxes), torch.cat(labels)
        dev = props.device
        keys = torch.rand(props.shape[0], generator=generator, device=dev if generator is None else generator.device).to(dev)
        gts = [getattr(g, 'tensor', g).to(dev) for g in gt_bboxes_3d]
        widths = {g.shape[1] for g in gts if g.shape[0]}
        if len(widths) > 1:
            _refuse(f"every sample's GT boxes must have the same width, got {sorted(widths)}", "GroupCorrectionHead")
        w = widths.pop() if widths else 7
        gt = torch.cat([g if g.shape[0] else g.new_zeros((0, w)) for g in gts]).float()
        gl = torch.cat([l.reshape(-1) for l in gt_labels_3d]).to(dev).long()
        inds, iou, gt_rows, glab, num_pos, num_rows = ops.roi_assign_sample(props, plab, [len(b) for b in boxes], keys, gt, gl,
                                                                            [g.shape[0] for g in gts], self.sample_cfg)
        batch_idx = torch.cat([torch.full((n,), b, dtype=torch.int64, device=dev) for b, n in enumerate(num_rows)])
        return RoiSampling(batch_idx, props[inds], iou, gt_rows, glab, gt, num_pos, num_rows)
