"""CenterHead (mmdet3d/models/dense_heads/centerpoint_head.py:240-830) on libsstb200: the reference's constructor keywords, forward
structure and state-dict keys; get_targets and the two losses run natively (ops.centerpoint_targets, ops.gaussian_focal_loss,
ops.centerpoint_l1_loss) with no host sync; get_bboxes is CenterPointBBoxCoder.decode
(core/bbox/coders/centerpoint_bbox_coders.py) and get_task_detections over ops.nms_gpu."""
import copy

import torch
from torch import nn

from . import ops
from .dcn_modules import ConvModule
from .registry import MODELS


def _gravity_boxes(boxes):
    """[N, 7|9] fp32 boxes with a gravity-centre z: from an object with `.tensor` / `.gravity_center` (LiDARInstance3DBoxes), or from a
    raw LiDAR tensor with a bottom-centre z (lidar_box3d.py:45-51: z + dz * 0.5)"""
    if hasattr(boxes, "gravity_center") and hasattr(boxes, "tensor"):
        return torch.cat((boxes.gravity_center, boxes.tensor[:, 3:]), dim=1)
    t = boxes
    z = t[:, 2:3] + t[:, 5:6] * 0.5
    return torch.cat((t[:, :2], z, t[:, 3:]), dim=1)


class CenterPointBBoxCoder:
    """core/bbox/coders/centerpoint_bbox_coders.py: decode only (top-K over the heatmap, boxes gathered at the K cells)."""

    def __init__(self, pc_range, out_size_factor, voxel_size, post_center_range=None, max_num=100, score_threshold=None, code_size=9,
                 type=None):
        self.pc_range, self.out_size_factor, self.voxel_size = pc_range, out_size_factor, voxel_size
        self.post_center_range, self.max_num, self.score_threshold, self.code_size = post_center_range, max_num, score_threshold, code_size

    @staticmethod
    def _gather_feat(feats, inds):
        return feats.gather(1, inds.unsqueeze(2).expand(inds.size(0), inds.size(1), feats.size(2)))

    def _transpose_and_gather_feat(self, feat, ind):
        feat = feat.permute(0, 2, 3, 1).contiguous()
        return self._gather_feat(feat.view(feat.size(0), -1, feat.size(3)), ind)

    def _topk(self, scores, K):
        batch, cat, height, width = scores.size()
        topk_scores, topk_inds = torch.topk(scores.view(batch, cat, -1), K)
        topk_inds = topk_inds % (height * width)
        topk_ys = (topk_inds.float() / torch.tensor(width, dtype=torch.float)).int().float()
        topk_xs = (topk_inds % width).int().float()
        topk_score, topk_ind = torch.topk(topk_scores.view(batch, -1), K)
        topk_clses = (topk_ind / torch.tensor(K, dtype=torch.float)).int()
        topk_inds = self._gather_feat(topk_inds.view(batch, -1, 1), topk_ind).view(batch, K)
        topk_ys = self._gather_feat(topk_ys.view(batch, -1, 1), topk_ind).view(batch, K)
        topk_xs = self._gather_feat(topk_xs.view(batch, -1, 1), topk_ind).view(batch, K)
        return topk_score, topk_inds, topk_clses, topk_ys, topk_xs

    def decode(self, heat, rot_sine, rot_cosine, hei, dim, vel, reg=None, task_id=-1):
        if self.post_center_range is None:
            raise NotImplementedError("Need to reorganize output as a batch, only support post_center_range is not None for now!")
        batch, K = heat.size(0), self.max_num
        scores, inds, clses, ys, xs = self._topk(heat, K)
        if reg is not None:
            reg = self._transpose_and_gather_feat(reg, inds).view(batch, K, 2)
            xs = xs.view(batch, K, 1) + reg[:, :, 0:1]
            ys = ys.view(batch, K, 1) + reg[:, :, 1:2]
        else:
            xs = xs.view(batch, K, 1) + 0.5
            ys = ys.view(batch, K, 1) + 0.5
        rot_sine = self._transpose_and_gather_feat(rot_sine, inds).view(batch, K, 1)
        rot_cosine = self._transpose_and_gather_feat(rot_cosine, inds).view(batch, K, 1)
        rot = torch.atan2(rot_sine, rot_cosine)
        hei = self._transpose_and_gather_feat(hei, inds).view(batch, K, 1)
        dim = self._transpose_and_gather_feat(dim, inds).view(batch, K, 3)
        clses = clses.view(batch, K).float()
        scores = scores.view(batch, K)
        xs = xs.view(batch, K, 1) * self.out_size_factor * self.voxel_size[0] + self.pc_range[0]
        ys = ys.view(batch, K, 1) * self.out_size_factor * self.voxel_size[1] + self.pc_range[1]
        parts = [xs, ys, hei, dim, rot]
        if vel is not None:
            parts.append(self._transpose_and_gather_feat(vel, inds).view(batch, K, 2))
        final_box_preds = torch.cat(parts, dim=2)
        pcr = torch.tensor(self.post_center_range, device=heat.device)
        mask = (final_box_preds[..., :3] >= pcr[:3]).all(2) & (final_box_preds[..., :3] <= pcr[3:]).all(2)
        if self.score_threshold is not None:
            thresh_mask = scores > self.score_threshold
        out = []
        for i in range(batch):
            cmask = mask[i, :]
            if self.score_threshold:
                cmask = cmask & thresh_mask[i]
            out.append(dict(bboxes=final_box_preds[i, cmask], scores=scores[i, cmask], labels=clses[i, cmask]))
        return out


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


@MODELS.register_module()
class CenterHead(nn.Module):
    """centerpoint_head.py:240-830.  forward(feats) -> a tuple over tasks of one-element lists of dicts {head name: [B, C, H, W]}.

    loss_cls must be GaussianFocalLoss and loss_bbox L1Loss, both with reduction 'mean' (the CenterHead configs' settings); anything else
    raises.  Unlike the reference, loss() leaves preds_dicts as it finds them: it neither overwrites preds_dicts[t][0]['heatmap'] with its
    clipped sigmoid nor adds an 'anno_box' entry.  gt boxes may be LiDARInstance3DBoxes-like objects (`.tensor`, `.gravity_center`) or
    raw [N, 7|9] LiDAR tensors with a bottom-centre z."""

    def __init__(self, in_channels=[128], tasks=None, train_cfg=None, test_cfg=None, bbox_coder=None, common_heads=dict(),
                 loss_cls=dict(type='GaussianFocalLoss', reduction='mean'), loss_bbox=dict(type='L1Loss', reduction='none', loss_weight=0.25),
                 separate_head=dict(type='SeparateHead', init_bias=-2.19, final_kernel=3), share_conv_channel=64, num_heatmap_convs=2,
                 conv_cfg=dict(type='Conv2d'), norm_cfg=dict(type='BN2d'), bias='auto', norm_bbox=True, init_cfg=None):
        assert init_cfg is None, 'To prevent abnormal initialization behavior, init_cfg is not allowed to be set'
        super().__init__()
        if loss_cls.get("type") != "GaussianFocalLoss" or loss_cls.get("reduction", "mean") != "mean":
            raise ValueError(f"CenterHead: loss_cls must be GaussianFocalLoss with reduction 'mean', got {loss_cls}")
        if loss_bbox.get("type") != "L1Loss" or loss_bbox.get("reduction", "mean") != "mean":
            raise ValueError(f"CenterHead: loss_bbox must be L1Loss with reduction 'mean', got {loss_bbox}")
        for name, cfg, defaults in (("loss_cls", loss_cls, dict(alpha=2.0, gamma=4.0)), ("loss_bbox", loss_bbox, {})):
            extra = {k: v for k, v in cfg.items() if k not in ("type", "reduction", "loss_weight") and defaults.get(k) != v}
            if extra:
                raise ValueError(f"CenterHead: {name} settings {extra} are not supported")
        num_classes = [len(t['class_names']) for t in tasks]
        self.class_names = [t['class_names'] for t in tasks]
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.in_channels, self.num_classes, self.norm_bbox = in_channels, num_classes, norm_bbox
        self.loss_cls_weight = float(loss_cls.get("loss_weight", 1.0))
        self.loss_bbox_weight = float(loss_bbox.get("loss_weight", 1.0))
        self.bbox_coder = CenterPointBBoxCoder(**bbox_coder) if bbox_coder is not None else None
        self.num_anchor_per_locs = [n for n in num_classes]
        self.fp16_enabled = False
        self.shared_conv = ConvModule(in_channels, share_conv_channel, kernel_size=3, padding=1, conv_cfg=conv_cfg, norm_cfg=norm_cfg,
                                      bias=bias)
        self.task_heads = nn.ModuleList()
        separate_head = copy.deepcopy(separate_head)
        for num_cls in num_classes:
            heads = copy.deepcopy(common_heads)
            heads.update(dict(heatmap=(num_cls, num_heatmap_convs)))
            separate_head.update(in_channels=share_conv_channel, heads=heads, num_cls=num_cls)
            self.task_heads.append(MODELS.build(separate_head))

    def init_weights(self):
        for head in self.task_heads:
            head.init_weights()

    def forward_single(self, x):
        x = self.shared_conv(x)
        return [task(x) for task in self.task_heads]

    def forward(self, feats):
        return tuple(map(list, zip(*[self.forward_single(x) for x in feats])))

    def get_targets(self, gt_bboxes_3d, gt_labels_3d):
        """Four lists over tasks: heatmaps [B, ncls, H, W], anno_boxes [B, max_objs, 10], inds [B, max_objs], masks [B, max_objs]."""
        cfg = self.train_cfg
        labels = [lab.long() for lab in gt_labels_3d]
        boxes = [_gravity_boxes(b).to(lab.device) for b, lab in zip(gt_bboxes_3d, labels)]
        dims = {b.shape[1] for b in boxes}
        if len(dims) != 1:
            raise ValueError(f"CenterHead.get_targets: every sample needs the same box width, got {sorted(dims)}")
        osf = cfg['out_size_factor']
        return ops.centerpoint_targets(torch.cat(boxes).float(), torch.cat(labels), [b.shape[0] for b in boxes], self.num_classes,
                                       cfg['point_cloud_range'][:2], cfg['voxel_size'][:2], osf,
                                       (cfg['grid_size'][0] // osf, cfg['grid_size'][1] // osf), cfg['gaussian_overlap'],
                                       cfg['min_radius'], cfg['max_objs'] * cfg['dense_reg'], self.norm_bbox)

    def loss(self, gt_bboxes_3d, gt_labels_3d, preds_dicts, **kwargs):
        """{'task{t}.loss_heatmap', 'task{t}.loss_bbox'}: the Gaussian focal loss of clip_sigmoid(heatmap) with avg_factor max(num_pos, 1),
        and the code-weighted L1 of the five regression heads at the targets' cells with avg_factor sum(mask) + 1e-4."""
        heatmaps, anno_boxes, inds, masks = self.get_targets(gt_bboxes_3d, gt_labels_3d)
        code_weights = self.train_cfg['code_weights']
        loss_dict = dict()
        for task_id, preds_dict in enumerate(preds_dicts):
            p = preds_dict[0]
            loss_heatmap, _ = ops.gaussian_focal_loss(p['heatmap'], heatmaps[task_id], self.loss_cls_weight)
            loss_bbox = ops.centerpoint_l1_loss(p, anno_boxes[task_id], inds[task_id], masks[task_id], code_weights, self.loss_bbox_weight)
            loss_dict[f'task{task_id}.loss_heatmap'] = loss_heatmap
            loss_dict[f'task{task_id}.loss_bbox'] = loss_bbox
        return loss_dict

    def get_bboxes(self, preds_dicts, img_metas, img=None, rescale=False):
        """[[bboxes, scores, labels] per sample]; bboxes are wrapped in img_metas[i]['box_type_3d'] when given, else a raw [N, 9] tensor
        with a bottom-centre z.  Rotated NMS only (nms_type 'circle' raises NotImplementedError)."""
        if self.test_cfg['nms_type'] != 'rotate':
            raise NotImplementedError(f"CenterHead.get_bboxes: nms_type {self.test_cfg['nms_type']!r}; only 'rotate' is implemented")
        rets = []
        for task_id, preds_dict in enumerate(preds_dicts):
            p = preds_dict[0]
            batch_dim = torch.exp(p['dim']) if self.norm_bbox else p['dim']
            temp = self.bbox_coder.decode(p['heatmap'].sigmoid(), p['rot'][:, 0].unsqueeze(1), p['rot'][:, 1].unsqueeze(1), p['height'],
                                          batch_dim, p.get('vel'), reg=p['reg'], task_id=task_id)
            rets.append(self.get_task_detections(self.num_classes[task_id], [b['scores'] for b in temp], [b['bboxes'] for b in temp],
                                                 [b['labels'] for b in temp], img_metas))
        ret_list = []
        for i in range(len(rets[0])):
            bboxes = torch.cat([ret[i]['bboxes'] for ret in rets])
            bboxes[:, 2] = bboxes[:, 2] - bboxes[:, 5] * 0.5
            meta = img_metas[i] if img_metas is not None else None
            if meta is not None and 'box_type_3d' in meta:
                bboxes = meta['box_type_3d'](bboxes, self.bbox_coder.code_size)
            scores = torch.cat([ret[i]['scores'] for ret in rets])
            flag, labels = 0, []
            for j, num_class in enumerate(self.num_classes):
                labels.append((rets[j][i]['labels'] + flag).int())
                flag += num_class
            ret_list.append([bboxes, scores, torch.cat(labels)])
        return ret_list

    def get_task_detections(self, num_class_with_bg, batch_cls_preds, batch_reg_preds, batch_cls_labels, img_metas):
        """centerpoint_head.py:703-830: per sample, rotated NMS over the BEV boxes (columns 0, 1, 3, 4, 6), then the post-centre range."""
        cfg = self.test_cfg
        post_center_range = cfg['post_center_limit_range']
        if len(post_center_range) > 0:
            post_center_range = torch.tensor(post_center_range, dtype=batch_reg_preds[0].dtype, device=batch_reg_preds[0].device)
        predictions_dicts = []
        for box_preds, cls_preds, cls_labels in zip(batch_reg_preds, batch_cls_preds, batch_cls_labels):
            top_scores = cls_preds.squeeze(-1)
            if num_class_with_bg == 1:
                top_labels = torch.zeros(cls_preds.shape[0], device=cls_preds.device, dtype=torch.long)
            else:
                top_labels = cls_labels.long()
            if cfg['score_threshold'] > 0.0:
                keep = top_scores >= torch.tensor([cfg['score_threshold']], device=cls_preds.device).type_as(cls_preds)
                top_scores, box_preds, top_labels = top_scores[keep], box_preds[keep], top_labels[keep]
            if top_scores.shape[0] != 0:
                boxes_for_nms = xywhr2xyxyr(box_preds[:, [0, 1, 3, 4, 6]])
                selected = ops.nms_gpu(boxes_for_nms, top_scores, thresh=cfg['nms_thr'], pre_maxsize=cfg['pre_max_size'],
                                       post_max_size=cfg['post_max_size'])
            else:
                selected = torch.zeros((0,), dtype=torch.long, device=box_preds.device)
            box_preds, top_labels, top_scores = box_preds[selected], top_labels[selected], top_scores[selected]
            if box_preds.shape[0] != 0:
                if post_center_range is not None:
                    mask = (box_preds[:, :3] >= post_center_range[:3]).all(1) & (box_preds[:, :3] <= post_center_range[3:]).all(1)
                    predictions_dicts.append(dict(bboxes=box_preds[mask], scores=top_scores[mask], labels=top_labels[mask]))
                else:
                    predictions_dicts.append(dict(bboxes=box_preds, scores=top_scores, labels=top_labels))
            else:
                dtype, device = batch_reg_preds[0].dtype, batch_reg_preds[0].device
                predictions_dicts.append(dict(bboxes=torch.zeros([0, self.bbox_coder.code_size], dtype=dtype, device=device),
                                              scores=torch.zeros([0], dtype=dtype, device=device),
                                              labels=torch.zeros([0], dtype=top_labels.dtype, device=device)))
        return predictions_dicts
