"""FSD's point segmentor: VoteSegHead (mmdet3d/models/decode_heads/segmentation_head.py) and VoteSegmentor
(mmdet3d/models/detectors/single_stage_fsd.py:155-392) on libsstb200.

VoteSegHead keeps the reference's constructor keywords, methods, loss-dict keys and state-dict keys (pre_seg_conv.* from build_mlp,
conv_seg and voting as nn.Linear).  Its MLP and the two Linears are plain torch (cuBLAS); its targets and losses run natively
(ops.voteseg_targets, ops.voteseg_loss) with no host sync.  VoteSegmentor composes the registered voxel encoder, middle encoder, backbone
and voxel-to-point neck around it."""
import torch
from torch import nn
from torch.utils.checkpoint import checkpoint

from . import ops
from .registry import MODELS

_FOCAL_KEYS = {"type", "use_sigmoid", "gamma", "alpha", "reduction", "loss_weight"}
_CE_KEYS = {"type", "use_sigmoid", "use_mask", "reduction", "class_weight", "loss_weight", "avg_non_ignore", "loss_name"}
_L1_KEYS = {"type", "reduction", "loss_weight"}


def _refuse(what):
    raise ValueError(f"VoteSegHead: {what}")


def _check_losses(loss_decode, loss_vote, loss_aux):
    if loss_aux is not None:
        _refuse(f"loss_aux is not supported, got {loss_aux}")
    d = dict(loss_decode)
    if d.get("reduction", "mean") != "mean":
        _refuse(f"loss_decode must reduce by 'mean', got {d.get('reduction')}")
    if d.get("type") == "FocalLoss":
        # explicit: the head reads a missing use_sigmoid as False (segmentation_head.py:57), mmdet's FocalLoss as True
        if d.get("use_sigmoid") is not True or set(d) - _FOCAL_KEYS:
            _refuse(f"FocalLoss needs an explicit use_sigmoid=True and no keys beyond {sorted(_FOCAL_KEYS)}, got {d}")
        if not float(d.get("gamma", 2.0)) >= 1.0:
            _refuse(f"FocalLoss gamma must be >= 1, got {d.get('gamma')}")
    elif d.get("type") == "CrossEntropyLoss":
        if d.get("use_sigmoid", False) or d.get("use_mask", False) or d.get("avg_non_ignore", False) or set(d) - _CE_KEYS:
            _refuse(f"CrossEntropyLoss needs use_sigmoid=False, use_mask=False, avg_non_ignore=False, got {d}")
        if d.get("class_weight") is not None and not isinstance(d["class_weight"], (list, tuple)):
            _refuse(f"CrossEntropyLoss class_weight must be a list, got {d['class_weight']!r}")
    else:
        _refuse(f"loss_decode must be a sigmoid FocalLoss or a softmax CrossEntropyLoss, got {d.get('type')}")
    v = dict(loss_vote)
    if v.get("type") != "L1Loss" or set(v) - _L1_KEYS or v.get("reduction", "mean") != "mean":
        _refuse(f"loss_vote must be L1Loss with reduction 'mean', got {v}")


@MODELS.register_module()
class VoteSegHead(nn.Module):
    """segmentation_head.py:15-283.  Differences from the reference, none of which changes a result:
    - get_targets and losses run natively: one launch for the batch's labels and vote targets, one fused pass for both losses and the
      training-log counts, no host round trip.
    - The reference's host-sync asserts in `losses` are dropped: `seg_label.max().item() == num_classes` (which requires a background
      point in the batch) and the range checks of the valid labels.  A label out of range makes the loss NaN instead.
    - A setting no config uses raises ValueError: loss_aux, a loss_decode other than FocalLoss with an explicit use_sigmoid=True and
      gamma >= 1 / softmax CrossEntropyLoss, a loss_vote other than L1Loss, and train_cfg with centroid_offset=True or extra_width."""

    def __init__(self, in_channel, num_classes, hidden_dims=[], dropout_ratio=0.5, conv_cfg=dict(type='Conv1d'),
                 norm_cfg=dict(type='naiveSyncBN1d'), act_cfg=dict(type='ReLU'),
                 loss_decode=dict(type='CrossEntropyLoss', use_sigmoid=False, class_weight=None, loss_weight=1.0),
                 loss_vote=dict(type='L1Loss'), loss_aux=None, ignore_index=255, logit_scale=1, checkpointing=False, init_bias=None,
                 init_cfg=None):
        super().__init__()
        _check_losses(loss_decode, loss_vote, loss_aux)
        end_channel = hidden_dims[-1] if len(hidden_dims) > 0 else in_channel
        self.channels, self.conv_cfg, self.norm_cfg, self.act_cfg = end_channel, conv_cfg, norm_cfg, act_cfg
        self.dropout_ratio, self.ignore_index = dropout_ratio, ignore_index
        self.use_sigmoid = loss_decode.get('use_sigmoid', False)
        self.bg_label = num_classes
        self.num_classes = num_classes if self.use_sigmoid else num_classes + 1
        # Base3DDecodeHead registers conv_seg first; the reference then replaces it with a Linear under the same name
        self.conv_seg = nn.Linear(end_channel, self.num_classes)
        self.dropout = nn.Dropout(dropout_ratio) if dropout_ratio > 0 else None
        self.pre_seg_conv = None
        if len(hidden_dims) > 0:
            self.pre_seg_conv = ops.build_mlp(in_channel, hidden_dims, norm_cfg, act=act_cfg['type'])
        self.voting = nn.Linear(end_channel, self.num_classes * 3)
        self.logit_scale = logit_scale
        self.fp16_enabled = False
        self.checkpointing = checkpointing
        self.init_bias = init_bias
        self.loss_aux = None
        self.loss_decode_cfg, self.loss_vote_cfg = dict(loss_decode), dict(loss_vote)
        self._train_cfg, self._loss_cfg = None, None
        self.test_cfg = None

    @property
    def train_cfg(self):
        return self._train_cfg

    @train_cfg.setter
    def train_cfg(self, cfg):
        if cfg is not None:
            if cfg.get('centroid_offset', False):
                _refuse("train_cfg centroid_offset=True is not supported")
            if cfg.get('extra_width', None) is not None:
                _refuse(f"train_cfg extra_width is not supported, got {cfg.get('extra_width')}")
        self._train_cfg, self._loss_cfg = cfg, None

    def init_weights(self):
        """lines 79-86 over decode_head.py:59-62: conv_seg normal(0, 0.01) with a zero bias, then the bias filled with init_bias"""
        nn.init.normal_(self.conv_seg.weight, 0, 0.01)
        nn.init.constant_(self.conv_seg.bias, 0)
        if self.init_bias is not None:
            self.conv_seg.bias.data.fill_(self.init_bias)

    def cls_seg(self, feat):
        if self.dropout is not None:
            feat = self.dropout(feat)
        return self.conv_seg(feat)

    def forward(self, voxel_feat):
        output = voxel_feat
        if self.pre_seg_conv is not None:
            if self.checkpointing:
                output = checkpoint(self.pre_seg_conv, voxel_feat, use_reentrant=True)
            else:
                output = self.pre_seg_conv(voxel_feat)
        logits = self.cls_seg(output)
        vote_preds = self.voting(output)
        return logits, vote_preds

    def loss_config(self):
        """the ops.VoteSegLossConfig of this head and its train_cfg (built once per train_cfg)"""
        if self._loss_cfg is None:
            d, cfg = self.loss_decode_cfg, self.train_cfg or {}
            thr = cfg.get('score_thresh', None)
            self._loss_cfg = ops.VoteSegLossConfig(
                self.num_classes, self.use_sigmoid, gamma=d.get('gamma', 2.0), alpha=d.get('alpha', 0.25),
                class_weight=d.get('class_weight'), logit_scale=self.logit_scale, loss_weight=d.get('loss_weight', 1.0),
                loss_weight_vote=self.loss_vote_cfg.get('loss_weight', 1.0), score_thresh=thr,
                class_names=cfg.get('class_names') if thr is not None else None,
                group_names=cfg.get('group_names') if thr is not None and not self.use_sigmoid else None)
        return self._loss_cfg

    def losses(self, seg_logit, vote_preds, seg_label, vote_targets, vote_mask):
        """lines 107-173: loss_sem_seg and loss_vote (fp32 device scalars with gradients), then the training-log recall_<name> (and
        num_fg for softmax heads) when train_cfg has score_thresh, as device tensors"""
        loss_sem_seg, loss_vote, metrics = ops.voteseg_loss(seg_logit, vote_preds, seg_label, vote_targets, vote_mask, self.loss_config())
        loss = dict(loss_sem_seg=loss_sem_seg, loss_vote=loss_vote)
        loss.update(metrics)
        return loss

    def forward_train(self, inputs, img_metas, pts_semantic_mask, vote_targets, vote_mask, return_preds=False):
        seg_logits, vote_preds = self.forward(inputs)
        losses = self.losses(seg_logits, vote_preds, pts_semantic_mask, vote_targets, vote_mask)
        if return_preds:
            return losses, dict(seg_logits=seg_logits, vote_preds=vote_preds)
        return losses

    def forward_test(self, inputs, img_metas, test_cfg):
        return self.forward(inputs)

    def get_targets(self, points_list, gt_bboxes_list, gt_labels_list):
        """lines 212-252 for the whole batch in one launch: (labels int64 [N], vote_targets [N, 3], vote_mask bool [N])"""
        return ops.voteseg_targets(list(points_list), None, gt_bboxes_list, gt_labels_list, self.bg_label)

    def encode_vote_targets(self, delta):
        return torch.sign(delta) * (delta.abs() ** 0.5)

    def decode_vote_targets(self, preds):
        return preds * preds.abs()


@MODELS.register_module()
class VoteSegmentor(nn.Module):
    """single_stage_fsd.py:155-392 over the registered modules.  voxel_layer is dynamic voxelisation (max_num_points=-1) through
    ops.Voxelization, run once over the concatenated batch.  The targets are computed from that concatenation too, so the points are
    concatenated once per step.  Unlike the reference, the tanh of `tanh_dims` is applied to a copy: the caller's point tensors are not
    modified in place."""

    def __init__(self, voxel_layer, voxel_encoder, middle_encoder, backbone, segmentation_head, decode_neck=None, auxiliary_head=None,
                 voxel_downsampling_size=None, train_cfg=None, test_cfg=None, init_cfg=None, pretrained=None, tanh_dims=None,
                 **extra_kwargs):
        super().__init__()
        if voxel_encoder['type'] != 'DynamicScatterVFE':
            raise ValueError(f"VoteSegmentor: the voxel encoder must be DynamicScatterVFE, got {voxel_encoder['type']}")
        if voxel_layer.get('max_num_points', -1) != -1:
            raise ValueError(f"VoteSegmentor: only dynamic voxelisation (max_num_points=-1) is supported, got {voxel_layer}")
        if decode_neck is None:
            raise ValueError("VoteSegmentor: decode_neck is required")
        self.voxel_layer = ops.Voxelization(**voxel_layer)
        self.voxel_encoder = MODELS.build(voxel_encoder)
        self.middle_encoder = MODELS.build(middle_encoder)
        self.backbone = MODELS.build(backbone)
        self.segmentation_head = MODELS.build(segmentation_head)
        self.segmentation_head.train_cfg = train_cfg
        self.segmentation_head.test_cfg = test_cfg
        self.decode_neck = MODELS.build(decode_neck)
        self.print_info = {}
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.cfg = train_cfg if train_cfg is not None else test_cfg
        self.num_classes = segmentation_head['num_classes']
        self.save_list = []
        self.point_cloud_range = voxel_layer['point_cloud_range']
        self.voxel_size = voxel_layer['voxel_size']
        self.voxel_downsampling_size = voxel_downsampling_size
        self.tanh_dims = tanh_dims
        self.use_multiscale_features = backbone.get('return_multiscale_features', False)

    @torch.no_grad()
    def voxelize(self, points):
        """(concatenated points, coors [N, 4] int32 = (sample, z, y, x)), as the reference's per-sample loop gives them"""
        batch_points = torch.cat(points, dim=0)
        coors = self.voxel_layer(batch_points)
        bidx = torch.cat([torch.full((p.shape[0], 1), i, dtype=coors.dtype, device=coors.device) for i, p in enumerate(points)])
        return batch_points, torch.cat([bidx, coors], 1)

    def extract_feat(self, points, img_metas):
        """lines 228-250"""
        batch_points, coors = self.voxelize(points)
        return self._extract(batch_points, coors.long())

    def _extract(self, batch_points, coors):
        voxel_features, voxel_coors, voxel2point_inds = self.voxel_encoder(batch_points, coors, return_inv=True)
        voxel_info = self.middle_encoder(voxel_features, voxel_coors)
        x = self.backbone(voxel_info)[0]
        padding = -1
        if 'shuffle_inds' not in voxel_info:
            voxel_feats_reorder = x['voxel_feats']
        else:
            voxel_feats_reorder = self.reorder(x['voxel_feats'], voxel_info['shuffle_inds'], voxel_info['voxel_keep_inds'], padding)
        out = self.decode_neck(batch_points, coors, voxel_feats_reorder, voxel2point_inds, padding)
        if self.use_multiscale_features:
            return out, coors, batch_points, x['decoder_features']
        return out, coors, batch_points

    def reorder(self, data, shuffle_inds, keep_inds, padding=-1):
        """lines 254-268: pad the dropped voxels and restore the voxel encoder's order"""
        num_voxel_no_drop = len(shuffle_inds)
        data_dim = data.size(1)
        temp_data = padding * data.new_ones((num_voxel_no_drop, data_dim))
        out_data = padding * data.new_ones((num_voxel_no_drop, data_dim))
        temp_data[keep_inds] = data
        out_data[shuffle_inds] = temp_data
        return out_data

    def voxel_downsample(self, points_list):
        """lines 270-281"""
        device = points_list[0].device
        out_points_list = []
        voxel_size = torch.tensor(self.voxel_downsampling_size, device=device)
        pc_range = torch.tensor(self.point_cloud_range, device=device)
        for points in points_list:
            coors = torch.div(points[:, :3] - pc_range[None, :3], voxel_size[None, :], rounding_mode='floor').long()
            out_points, new_coors = ops.scatter_v2(points, coors, mode='avg', return_inv=False)
            out_points_list.append(out_points)
        return out_points_list

    def _prepare(self, points):
        if self.tanh_dims is not None:
            if len(self.tanh_dims) > 0:
                out = []
                for p in points:
                    p = p.clone()
                    p[:, self.tanh_dims] = torch.tanh(p[:, self.tanh_dims])
                    out.append(p)
                points = out
        elif points[0].size(1) in (4, 5):
            # the reference's way of scaling the intensity and elongation of Waymo points
            points = [torch.cat([p[:, :3], torch.tanh(p[:, 3:])], dim=1) for p in points]
        if self.voxel_downsampling_size is not None:
            points = self.voxel_downsample(points)
        return points

    def forward_train(self, points, img_metas, gt_bboxes_3d, gt_labels_3d, as_subsegmentor=False):
        """lines 283-342"""
        points = self._prepare(points)
        batch_points, coors = self.voxelize(points)
        offsets = [0]
        for p in points:
            offsets.append(offsets[-1] + p.shape[0])
        labels, vote_targets, vote_mask = ops.voteseg_targets(batch_points, offsets, gt_bboxes_3d, gt_labels_3d,
                                                              self.segmentation_head.bg_label)
        if self.use_multiscale_features:
            neck_out, pts_coors, points, decoder_features = self._extract(batch_points, coors.long())
        else:
            neck_out, pts_coors, points = self._extract(batch_points, coors.long())
            decoder_features = None
        losses = dict()
        feats = neck_out[0]
        valid_pts_mask = neck_out[1]
        points = points[valid_pts_mask]
        pts_coors = pts_coors[valid_pts_mask]
        labels = labels[valid_pts_mask]
        vote_targets = vote_targets[valid_pts_mask]
        vote_mask = vote_mask[valid_pts_mask]
        assert feats.size(0) == labels.size(0)
        if as_subsegmentor:
            loss_decode, preds_dict = self.segmentation_head.forward_train(feats, img_metas, labels, vote_targets, vote_mask,
                                                                           return_preds=True)
            losses.update(loss_decode)
            offsets = self.segmentation_head.decode_vote_targets(preds_dict['vote_preds'])
            return dict(seg_points=points, seg_logits=preds_dict['seg_logits'], seg_vote_preds=preds_dict['vote_preds'], offsets=offsets,
                        seg_feats=feats, batch_idx=pts_coors[:, 0], losses=losses, decoder_features=decoder_features)
        loss_decode = self.segmentation_head.forward_train(feats, img_metas, labels, vote_targets, vote_mask, return_preds=False)
        losses.update(loss_decode)
        return losses

    def simple_test(self, points, img_metas, gt_bboxes_3d=None, gt_labels_3d=None, rescale=False):
        """lines 345-386"""
        points = self._prepare(points)
        if self.use_multiscale_features:
            x, pts_coors, points, decoder_features = self.extract_feat(points, img_metas)
        else:
            x, pts_coors, points = self.extract_feat(points, img_metas)
            decoder_features = None
        feats = x[0]
        valid_pts_mask = x[1]
        points = points[valid_pts_mask]
        pts_coors = pts_coors[valid_pts_mask]
        seg_logits, vote_preds = self.segmentation_head.forward_test(feats, img_metas, self.test_cfg)
        offsets = self.segmentation_head.decode_vote_targets(vote_preds)
        return dict(seg_points=points, seg_logits=seg_logits, seg_vote_preds=vote_preds, offsets=offsets, seg_feats=feats,
                    batch_idx=pts_coors[:, 0], decoder_features=decoder_features)
