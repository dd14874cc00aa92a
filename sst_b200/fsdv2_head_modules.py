"""FSDv2's detection head: FSDV2Head (mmdet3d/models/dense_heads/fsd_v2_head.py) on libsstb200.

The head shares SparseClusterHeadV2's MLPs, state-dict keys (shared_mlp.*, task_heads.{i}.{center,dim,rot,vel,score}.*), fused targets
and losses and segmented-NMS proposals (cluster_head_modules._ClusterHeadBase) and adds what the FSDv2 configs need: the in-box test on
each virtual voxel's point centroid (train_cfg centroid_assign, `aux_xyz`), code size 10 with velocity targets and loss_vel (nuScenes),
task class lists in any order relative to class_names, and test_cfg all_task_max_num."""
import torch

from .cluster_head_modules import _ClusterHeadBase, _check_losses, _refuse
from .registry import MODELS

_NAME = "FSDV2Head"


@MODELS.register_module()
class FSDV2Head(_ClusterHeadBase):
    """fsd_v2_head.py:17-591.  Differences from the reference, beyond SparseClusterHeadV2's (cluster_head_modules.py: one targets
    launch and one fused loss for every task and sample with no host sync, dropped `.item()` asserts, NaN for an out-of-range batch
    index in `loss`, at most two host syncs in get_bboxes):
    - The paste-flag asserts of get_targets_single (`pos_gt_bboxes[:, 9].max().item() in (0, 1)`) are dropped: column 9 is the
      velocity weight as it is.  Every sample with GTs must give them the same width, 9 or 10, for code size 10.
    - loss_vel is the same L1 / SmoothL1 element as the other box losses, times the flag, over 2 * num_pos (the local count: the
      reference calls it without avg_factor); exactly 0 for a task without a local positive.
    - get_bboxes cuts every sample over all_task_max_num with one batched topk; its boxes are [N, 9] for code size 10, also for a sample
      without clusters, where the reference gives [0, 7].
    - print_info[f'n_pos_t{t}'] is a [1] device tensor, set without a host sync.
    - `loss` with train_cfg centroid_assign and no aux_xyz raises ValueError (the reference asserts).
    - A setting no config uses raises ValueError: loss_iou / iou_mlp, corner_loss_cfg, enlarge_width, a code size other than 8 / 10,
      code size 10 without loss_vel or without a `vel` attribute (and loss_vel with code size 8), a loss_cls other than a sigmoid
      FocalLoss with gamma >= 1, box losses other than L1Loss / SmoothL1Loss with reduction 'mean' (loss_vel included, all of one type
      and beta), task class lists that are not a permutation of class_names, and train_cfg with assign_by_dist, max_assign_dist or
      code_weight.  get_bboxes raises ValueError for nms_pre > 0 or a per-class nms_thr list."""
    _NAME = _NAME
    _LOG_NUM_POS = True
    _TOPK = True

    def __init__(self, num_classes, bbox_coder, loss_cls, loss_center, loss_size, loss_rot, in_channel, shared_mlp_dims, tasks, class_names,
                 common_attrs, num_cls_layer, cls_hidden_dim, separate_head, cls_mlp=None, reg_mlp=None, iou_mlp=None, train_cfg=None,
                 test_cfg=None, norm_cfg=dict(type='LN'), loss_iou=None, act='relu', corner_loss_cfg=None, enlarge_width=None,
                 as_rpn=False, init_cfg=None, shared_dropout=0, loss_vel=None):
        super().__init__()
        if loss_iou is not None or iou_mlp is not None:
            _refuse("loss_iou / iou_mlp are not supported", _NAME)
        if corner_loss_cfg is not None:
            _refuse("corner_loss_cfg is not supported", _NAME)
        if enlarge_width is not None:
            _refuse("enlarge_width is not supported", _NAME)
        coder = dict(bbox_coder)
        code = coder.get("code_size", 8)
        if coder.get("type") != "BasePointBBoxCoder" or code not in (8, 10):
            _refuse(f"bbox_coder must be BasePointBBoxCoder with code_size 8 or 10, got {coder}", _NAME)
        if (code == 10) != (loss_vel is not None):
            _refuse(f"code_size 10 goes with loss_vel and code_size 8 without it, got code_size {code} and loss_vel {loss_vel}", _NAME)
        if code == 10 and 'vel' not in common_attrs:
            _refuse(f"code_size 10 needs a 'vel' attribute in common_attrs, got {sorted(common_attrs)}", _NAME)
        regs = dict(loss_center=loss_center, loss_size=loss_size, loss_rot=loss_rot)
        if loss_vel is not None:
            regs['loss_vel'] = loss_vel
        _check_losses(loss_cls, regs, _NAME)
        all_names = []
        for t in tasks:
            all_names += t['class_names']
        if sorted(all_names) != sorted(class_names):          # "the order does not matter" (line 98)
            _refuse(f"the tasks' class names {all_names} must be a permutation of class_names {list(class_names)}", _NAME)
        self._build(num_classes, class_names, tasks, in_channel, shared_mlp_dims, norm_cfg, act, shared_dropout, common_attrs,
                    num_cls_layer, cls_hidden_dim, separate_head, train_cfg, test_cfg, as_rpn, loss_cls, loss_center, loss_size, loss_rot,
                    code_size=code, loss_vel=loss_vel)

    def _assign_xyz(self, aux_xyz):
        """lines 359-362: the points of the in-box test, aux_xyz under train_cfg centroid_assign, else the voxel centres"""
        if not (self.train_cfg or {}).get('centroid_assign', False):
            return None
        if aux_xyz is None:
            _refuse("train_cfg centroid_assign needs aux_xyz (the virtual voxels' centroids)", _NAME)
        return aux_xyz

    def loss(self, cls_logits, reg_preds, voxel_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d, img_metas=None, iou_logits=None,
             gt_bboxes_ignore=None, aux_xyz=None):
        """lines 134-165: every task's loss_single_task in one targets launch and one fused loss; no host sync"""
        assert isinstance(cls_logits, list) and isinstance(reg_preds, list)
        assert len(cls_logits) == len(reg_preds) == len(self.tasks)
        return self._losses(list(range(len(self.tasks))), cls_logits, reg_preds, voxel_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d,
                            self._assign_xyz(aux_xyz))

    def loss_single_task(self, task_id, cls_logits, reg_preds, voxel_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d, iou_logits=None,
                         aux_xyz=None):
        """lines 168-275 for one task"""
        return self._losses([task_id], [cls_logits], [reg_preds], voxel_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d,
                            self._assign_xyz(aux_xyz))

    def get_targets(self, num_task_classes, voxel_xyz, batch_idx, gt_bboxes_3d, gt_labels_3d, reg_preds=None, aux_xyz=None):
        """lines 306-395 for GTs whose labels are already within the task (modify_gt_for_single_task): (labels, label_weights,
        bbox_targets [M, code_size], bbox_weights [M, code_size], None) over the whole batch, from one launch.  For code size 10 the
        weights' velocity columns are the positives' copy-paste flag (1 for 9-column GTs)."""
        return self._targets_one_task(num_task_classes, voxel_xyz, batch_idx, gt_bboxes_3d, gt_labels_3d, self._assign_xyz(aux_xyz))

    @torch.no_grad()
    def get_bboxes(self, cls_logits, reg_preds, voxel_xyz, cluster_inds, input_metas, iou_logits=None, rescale=False):
        """lines 415-474 for the whole batch: per sample, the (boxes, scores, global labels) of every task in task order, boxes [N, 7]
        or, for code size 10, [N, 9] with the velocity; then, with test_cfg all_task_max_num, each sample over it cut to its top-scoring
        boxes by one batched topk.  One segmented NMS for every (sample, task, class); no host sync beyond the NMS's."""
        return super().get_bboxes(cls_logits, reg_preds, voxel_xyz, cluster_inds, input_metas, iou_logits, rescale)
