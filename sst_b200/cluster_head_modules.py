"""FSD's first-stage detection head: FSDSeparateHead and SparseClusterHeadV2 (mmdet3d/models/dense_heads/sparse_cluster_head{,_v2}.py)
on libsstb200.

The MLPs are ops.build_mlp (torch / cuBLAS) under the reference's state-dict keys (shared_mlp.*, task_heads.{i}.{center,dim,rot,score}.*).
The targets of every task and sample run in one launch (ops.cluster_head_targets) and the losses of every task in one fused launch
sequence (ops.cluster_head_loss), with no host sync.  get_bboxes decodes every task with the reference's own torch ops and runs every
(sample, task, class) as a segment of one segmented NMS (ops.multiclass_nms_groups).  _ClusterHeadBase holds what SparseClusterHeadV2
shares with FSDV2Head (fsdv2_head_modules.py)."""
import copy

import torch
import torch.distributed as dist
from torch import nn

from . import ops
from .anchor3d_modules import xywhr2xyxyr
from .registry import MODELS

_FOCAL_KEYS = {"type", "use_sigmoid", "gamma", "alpha", "reduction", "loss_weight"}
_REG_KEYS = {"L1Loss": {"type", "reduction", "loss_weight"}, "SmoothL1Loss": {"type", "reduction", "loss_weight", "beta"}}
_EPS = 1e-6   # BasePointBBoxCoder.EPS


def _refuse(what, name="SparseClusterHeadV2"):
    raise ValueError(f"{name}: {what}")


def reduce_mean(tensor):
    """mmdet 2.14 reduce_mean: divide by the world size, then all_reduce SUM; the identity without a process group.  No host sync."""
    if not (dist.is_available() and dist.is_initialized()):
        return tensor
    tensor = tensor.clone()
    dist.all_reduce(tensor.div_(dist.get_world_size()), op=dist.ReduceOp.SUM)
    return tensor


def _check_losses(loss_cls, regs, head="SparseClusterHeadV2"):
    c = dict(loss_cls)
    if c.get("type") != "FocalLoss" or not c.get("use_sigmoid", True) or set(c) - _FOCAL_KEYS or c.get("reduction", "mean") != "mean":
        _refuse(f"loss_cls must be a sigmoid FocalLoss with reduction 'mean', got {c}", head)
    if not float(c.get("gamma", 2.0)) >= 1.0:
        _refuse(f"FocalLoss gamma must be >= 1, got {c.get('gamma')}", head)
    kinds = set()
    for name, r in regs.items():
        d = dict(r)
        if d.get("type") not in _REG_KEYS or set(d) - _REG_KEYS[d["type"]] or d.get("reduction", "mean") != "mean":
            _refuse(f"{name} must be L1Loss or SmoothL1Loss with reduction 'mean', got {d}", head)
        kinds.add((d["type"], float(d.get("beta", 1.0)) if d["type"] == "SmoothL1Loss" else None))
    if len(kinds) != 1:
        names = list(regs)
        _refuse(f"{', '.join(names[:-1])} and {names[-1]} must share their type and beta, got {sorted(kinds, key=str)}", head)


def decode(reg_preds, base_points):
    """BasePointBBoxCoder.decode with the reference's torch ops: [N, 7] (xyz, dims, yaw) bottom-centre boxes for code size 8, [N, 9]
    with the velocity columns appended for code size 10"""
    xyz = reg_preds[:, :3] + base_points
    dims = reg_preds[:, 3:6].exp() - _EPS
    yaw = torch.atan2(reg_preds[:, 6:7], reg_preds[:, 7:8])
    if reg_preds.shape[1] == 10:
        return torch.cat([xyz, dims, yaw, reg_preds[:, 8:10]], dim=1)
    return torch.cat([xyz, dims, yaw], dim=1)


@MODELS.register_module()
class FSDSeparateHead(nn.Module):
    """sparse_cluster_head_v2.py:17-41: one build_mlp per attribute, (out_dim, num_layer, hidden_dim) each"""

    def __init__(self, in_channels, attrs, norm_cfg=dict(type='LN'), act='relu', init_cfg=None):
        super().__init__()
        self.attrs = attrs
        for attr_name in self.attrs:
            out_dim, num_layer, hidden_dim = self.attrs[attr_name]
            self.__setattr__(attr_name, ops.build_mlp(in_channels, [hidden_dim] * num_layer + [out_dim], norm_cfg, is_head=True, act=act))

    def forward(self, x):
        return {attr_name: self.__getattr__(attr_name)(x) for attr_name in self.attrs}


class _ClusterHeadBase(nn.Module):
    """What SparseClusterHeadV2 and FSDV2Head share: the MLPs and their state-dict keys, the train_cfg refusals, the forward, the fused
    targets and losses of every task, modify_gt_for_single_task, and get_bboxes over one segmented NMS.  A subclass sets _NAME, calls
    _build, and may set _LOG_NUM_POS (print_info's n_pos_t{t}) and _TOPK (test_cfg all_task_max_num)."""
    _NAME = "SparseClusterHeadV2"
    _LOG_NUM_POS = False
    _TOPK = False

    def _build(self, num_classes, class_names, tasks, in_channel, shared_mlp_dims, norm_cfg, act, shared_dropout, common_attrs,
               num_cls_layer, cls_hidden_dim, separate_head, train_cfg, test_cfg, as_rpn, loss_cls, loss_center, loss_size, loss_rot,
               code_size=8, loss_vel=None):
        self.num_classes, self.class_names, self.tasks = num_classes, list(class_names), tasks
        self.box_code_size = code_size
        self.as_rpn, self.corner_loss_cfg, self.enlarge_width, self.loss_iou, self.loss_vel = as_rpn, None, None, None, None
        self.loss_cls_cfg, self.loss_reg_cfgs = dict(loss_cls), (dict(loss_center), dict(loss_size), dict(loss_rot))
        self.shared_mlp = None
        if len(shared_mlp_dims) > 0:
            self.shared_mlp = ops.build_mlp(in_channel, shared_mlp_dims, norm_cfg, act=act, dropout=shared_dropout)
        self.conv_cls = None
        self.conv_reg = None
        sep_in = shared_mlp_dims[-1] if self.shared_mlp is not None else in_channel
        self.task_heads = nn.ModuleList()
        separate_head = dict(separate_head)
        for t in tasks:
            attrs = copy.deepcopy(common_attrs)
            attrs.update(dict(score=(len(t['class_names']), num_cls_layer, cls_hidden_dim)))
            self.task_heads.append(MODELS.build(dict(separate_head, in_channels=sep_in, attrs=attrs)))
        self.fp16_enabled = False
        self.print_info = {}
        self.save_list = []
        self._train_cfg, self.test_cfg = None, test_cfg
        self.sync_reg_avg_factor = self.sync_cls_avg_factor = False
        self.train_cfg = train_cfg
        reg = self.loss_reg_cfgs[0]
        vel = {} if loss_vel is None else dict(loss_weight_vel=loss_vel.get('loss_weight', 1.0))
        self.loss_config = ops.ClusterHeadLossConfig(
            gamma=loss_cls.get('gamma', 2.0), alpha=loss_cls.get('alpha', 0.25), loss_weight_cls=loss_cls.get('loss_weight', 1.0),
            loss_weight_center=loss_center.get('loss_weight', 1.0), loss_weight_size=loss_size.get('loss_weight', 1.0),
            loss_weight_rot=loss_rot.get('loss_weight', 1.0), smooth_l1=reg['type'] == 'SmoothL1Loss', beta=reg.get('beta', 1.0), **vel)

    @property
    def train_cfg(self):
        return self._train_cfg

    @train_cfg.setter
    def train_cfg(self, cfg):
        if cfg is not None:
            for k in ('assign_by_dist', 'max_assign_dist', 'code_weight'):
                if cfg.get(k, None) not in (None, False):
                    _refuse(f"train_cfg {k} is not supported, got {cfg.get(k)}", self._NAME)
        self._train_cfg = cfg
        self.sync_reg_avg_factor = False if cfg is None else cfg.get('sync_reg_avg_factor', True)
        self.sync_cls_avg_factor = False if cfg is None else cfg.get('sync_cls_avg_factor', False)

    def forward(self, feats, pts_xyz=None, pts_inds=None):
        if self.shared_mlp is not None:
            feats = self.shared_mlp(feats)
        cls_logit_list, reg_pred_list = [], []
        for h in self.task_heads:
            ret = h(feats)
            cls_logit_list.append(ret['score'])
            reg = [ret['center'], ret['dim'], ret['rot']] + ([ret['vel']] if 'vel' in ret else [])
            reg_pred_list.append(torch.cat(reg, dim=-1))
        return dict(cls_logits=cls_logit_list, reg_preds=reg_pred_list)

    def _task_names(self, task_ids):
        return [self.tasks[i]['class_names'] for i in task_ids]

    def _losses(self, task_ids, cls_logits, reg_preds, cluster_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d, assign_xyz=None):
        labels, targets, num_pos = ops.cluster_head_targets(cluster_xyz.float(), cluster_inds, gt_bboxes_3d, gt_labels_3d,
                                                            self._task_names(task_ids), self.class_names,
                                                            assign_xyz=None if assign_xyz is None else assign_xyz.float(),
                                                            code_size=self.box_code_size)
        T, M = len(task_ids), cluster_xyz.shape[0]
        cls_avg = torch.full((T,), float(M), dtype=torch.float32, device=cluster_xyz.device)
        if self.sync_cls_avg_factor:
            cls_avg = reduce_mean(cls_avg)
        reg_avg = num_pos.float()
        if self.sync_reg_avg_factor:
            reg_avg = reduce_mean(reg_avg)
        losses = ops.cluster_head_loss(cls_logits, reg_preds, labels, targets, num_pos, cls_avg, reg_avg, self.loss_config)
        names = ('loss_cls', 'loss_center', 'loss_size', 'loss_rot') + (('loss_vel',) if self.box_code_size == 10 else ())
        out = {}
        for k, t in enumerate(task_ids):
            for q, name in enumerate(names):
                out[f'{name}.task{t}'] = losses[k, q]
        if self._LOG_NUM_POS:
            n = num_pos.float()
            for k, t in enumerate(task_ids):
                self.print_info[f'n_pos_t{t}'] = n[k:k + 1]
        return out

    def modify_gt_for_single_task(self, gt_bboxes_3d, gt_labels_3d, task_id):
        """v2 lines 299-326: per sample, the task's GTs class by class in the task's order, labels renumbered within the task"""
        out_b, out_l = [], []
        for boxes, labels in zip(gt_bboxes_3d, gt_labels_3d):
            if labels.numel() == 0:
                out_b.append(boxes)
                out_l.append(labels)
                continue
            sel, lab = [], []
            for i, name in enumerate(self.tasks[task_id]['class_names']):
                m = labels == self.class_names.index(name)
                sel.append(boxes[m])
                lab.append(torch.full_like(labels[m], i))
            # a box object (LiDARInstance3DBoxes) concatenates through its own `cat`, as in the reference; a raw tensor through torch
            out_b.append(boxes.cat(sel) if hasattr(boxes, 'cat') and not isinstance(boxes, torch.Tensor) else torch.cat(sel))
            out_l.append(torch.cat(lab))
        return out_b, out_l

    def _targets_one_task(self, num_task_classes, cluster_xyz, batch_idx, gt_bboxes_3d, gt_labels_3d, assign_xyz=None):
        """get_targets for GTs whose labels are already within the task (modify_gt_for_single_task): (labels, label_weights,
        bbox_targets, bbox_weights, None) over the whole batch, from one launch"""
        names = list(range(num_task_classes))
        code = self.box_code_size
        labels, targets, _ = ops.cluster_head_targets(cluster_xyz.float(), batch_idx, gt_bboxes_3d, gt_labels_3d, [names], names,
                                                      assign_xyz=None if assign_xyz is None else assign_xyz.float(), code_size=code)
        labels, targets = labels[0], targets[0]
        pos = ((labels >= 0) & (labels < num_task_classes)).float()
        weights = pos[:, None].expand(-1, code).contiguous()
        if code == 10:                # the velocity columns carry the copy-paste flag (the targets' column 10, 0 off the positives)
            weights[:, 8:] = torch.where(pos[:, None] > 0, targets[:, 10:], torch.zeros_like(targets[:, 10:]))
            targets = targets[:, :code].contiguous()
        return labels, torch.ones_like(pos), targets, weights, None

    def split_by_batch(self, data, batch_idx, batch_size):
        """sparse_cluster_head.py:269-278 without the `.item()` assert"""
        if batch_size == 1:
            return [data]
        return [data[batch_idx == i] for i in range(batch_size)]

    def combine_by_batch(self, data_list, batch_idx, batch_size):
        """sparse_cluster_head.py:280-289"""
        assert len(data_list) == batch_size
        if data_list[0] is None:
            return None
        full = data_list[0].new_zeros((len(batch_idx),) + data_list[0].shape[1:])
        for i, data in enumerate(data_list):
            full[batch_idx == i] = data
        return full

    def _global_labels(self, dev):
        """per task, the global class id of each of its classes, on `dev` (copied to the device once)"""
        cache = self.__dict__.setdefault('_glob', {})
        if dev not in cache:
            cache[dev] = [torch.tensor([self.class_names.index(n) for n in t['class_names']], dtype=torch.long, device=dev)
                          for t in self.tasks]
        return cache[dev]

    @torch.no_grad()
    def get_bboxes(self, cls_logits, reg_preds, cluster_xyz, cluster_inds, input_metas, iou_logits=None, rescale=False):
        """v2 lines 415-576 for the whole batch: per sample, the (boxes, scores, global labels) of every task in task order, each task's
        boxes in box3d_multiclass_nms's order.  Sigmoid, decode and xywhr2xyxyr are the reference's torch ops over every task at once;
        every (sample, task, class) is one segment of one segmented NMS."""
        assert len(cls_logits) == len(reg_preds) == len(self.tasks)
        if self.as_rpn:
            cfg = self.train_cfg['rpn'] if self.training else self.test_cfg['rpn']
        else:
            cfg = self.test_cfg
        if cfg.get('nms_pre', -1) > 0:
            _refuse(f"get_bboxes with nms_pre > 0 is not supported, got {cfg.get('nms_pre')}", self._NAME)
        nms_thr = cfg['nms_thr']
        if isinstance(nms_thr, (list, tuple)):
            _refuse(f"get_bboxes with a per-class nms_thr is not supported, got {nms_thr}", self._NAME)
        B, T = len(input_metas), len(self.tasks)
        xyz = cluster_xyz.float()
        M, dev = xyz.shape[0], xyz.device
        bidx = cluster_inds if cluster_inds.ndim == 1 else cluster_inds[:, 1]
        counts = [len(t['class_names']) for t in self.tasks]
        Cmax = max(counts)
        boxes = decode(torch.cat([r.float() for r in reg_preds]), xyz[:, :3].repeat(T, 1))
        box_dim = boxes.shape[1]
        # LiDAR bev = columns (0, 1, 3, 4, 6), stacked rather than list-indexed: a list index is a host-to-device copy, a host sync
        boxes_for_nms = xywhr2xyxyr(torch.stack([boxes[:, 0], boxes[:, 1], boxes[:, 3], boxes[:, 4], boxes[:, 6]], 1))
        score_thr = cfg.get('score_thr', 0)
        if B == 1:                 # split_by_batch returns every cluster for a batch of one, whatever its index
            bidx = torch.zeros_like(bidx)
        valid = (bidx >= 0) & (bidx < B)
        cls, idx, sc, grp = [], [], [], []
        rows = torch.arange(M, device=dev)
        for t, x in enumerate(cls_logits):
            s = x.float().sigmoid()
            C = counts[t]
            c = torch.arange(C * M, device=dev) // M                      # class-major, input order within a class
            r = rows.repeat(C)
            v = s.t().reshape(-1)
            g = torch.where(valid[r] & (v > score_thr), bidx[r] * T + t, torch.full_like(r, B * T))
            cls.append(c), idx.append(r + t * M), sc.append(v), grp.append(g)
        res = ops.multiclass_nms_groups(boxes, boxes_for_nms, torch.cat(cls), torch.cat(idx), torch.cat(sc), torch.cat(grp), B * T, Cmax,
                                        [nms_thr] * Cmax, cfg['max_num'], cfg['use_rotate_nms'])
        glob = self._global_labels(dev)
        out = []
        for b in range(B):
            bb, ss, ll = [], [], []
            for t in range(T):
                r = res[b * T + t]
                if r is None:
                    continue
                bb.append(r[0]), ss.append(r[1]), ll.append(glob[t][r[2]])
            ob = torch.cat(bb) if bb else xyz.new_zeros((0, box_dim))
            os_ = torch.cat(ss) if ss else xyz.new_zeros((0,))
            ol = torch.cat(ll) if ll else torch.zeros((0,), dtype=torch.long, device=dev)
            out.append((ob, os_, ol))
        if self._TOPK:
            out = _all_task_topk(out, (self.test_cfg or {}).get('all_task_max_num', None))
        for b in range(B):
            ob, os_, ol = out[b]
            meta = input_metas[b]
            if meta is not None and 'box_type_3d' in meta:
                out[b] = (meta['box_type_3d'](ob, ob.size(1)), os_, ol)
        return out


def _all_task_topk(results, k):
    """fsd_v2_head.py:459-472: per sample with more than k boxes over all tasks, its k top-scoring boxes in descending score.  The
    samples to cut are known from the host-side box counts; their scores go into one [n, N_max] -inf-padded matrix for one batched
    topk.  No host sync."""
    if k is None:
        return results
    cut = [b for b, r in enumerate(results) if r[1].shape[0] > k]
    if not cut:
        return results
    n = [results[b][1].shape[0] for b in cut]
    pad = results[cut[0]][1].new_full((len(cut), max(n)), float('-inf'))
    for i, b in enumerate(cut):
        pad[i, :n[i]] = results[b][1]
    top = pad.topk(k, dim=1).indices
    results = list(results)
    for i, b in enumerate(cut):
        results[b] = tuple(a[top[i]] for a in results[b])
    return results


@MODELS.register_module()
class SparseClusterHeadV2(_ClusterHeadBase):
    """sparse_cluster_head_v2.py:44-576 over sparse_cluster_head.py.  Differences from the reference:
    - The targets of every task and sample come from one launch, and the losses of every task from one fused launch sequence; `loss`
      makes no host round trip.  get_bboxes runs every (sample, task, class) in one segmented NMS with at most two host syncs in all
      (the candidate counts, then, when the cfg has an nms_thr, the kept counts: the training `rpn` cfg, nms_thr None, makes only the
      first) instead of box3d_multiclass_nms's per (task, sample).
    - The host-sync asserts are dropped: `batch_idx.max().item() + 1 <= batch_size` in split_by_batch,
      `out_labels.max().item() < num_classes_this_task` and `(gt_labels_3d >= 0).all()` in modify_gt_for_single_task, and
      `(label_weights == 1).all()`.  A GT with a negative label, or of a class in no task, takes part in no task instead of failing the
      assert.
    - In `loss`, a cluster whose batch index is outside [0, B) gets label -1 and NaN targets, so loss_cls is NaN.  The reference asserts
      on an index >= B in training mode (split_by_batch) and otherwise leaves such a cluster a class-0 row of zeros for B > 1.
    - In get_bboxes, with B > 1 a cluster whose batch index is outside [0, B) is dropped, as the reference's boolean split drops it in
      eval mode (in training mode the reference asserts on an index >= B); with B = 1 every cluster belongs to the one sample, as
      split_by_batch returns every row for a batch of one.
    - get_bboxes returns int64 labels for a sample without clusters; the reference returns a float zeros(0) there
      (`reg_preds.new_zeros(0)`).
    - The focal loss is the stable softplus form of mmdet's py_sigmoid_focal_loss, exact at any logit; mmcv's CUDA kernel, which the
      reference reaches on the GPU, clamps its log and saturates near 87 for logits beyond about +-17.
    - A setting no config uses raises ValueError: loss_iou / iou_mlp, corner_loss_cfg, enlarge_width, loss_vel, a code size other than
      8, a loss_cls other than a sigmoid FocalLoss with gamma >= 1, box losses other than L1Loss / SmoothL1Loss with reduction 'mean'
      (all three of one type and beta), and train_cfg with assign_by_dist, max_assign_dist or code_weight.  get_bboxes raises
      ValueError for nms_pre > 0 or a per-class nms_thr list."""

    def __init__(self, num_classes, bbox_coder, loss_cls, loss_center, loss_size, loss_rot, in_channel, shared_mlp_dims, tasks, class_names,
                 common_attrs, num_cls_layer, cls_hidden_dim, separate_head, cls_mlp=None, reg_mlp=None, iou_mlp=None, train_cfg=None,
                 test_cfg=None, norm_cfg=dict(type='LN'), loss_iou=None, act='relu', corner_loss_cfg=None, enlarge_width=None,
                 as_rpn=False, init_cfg=None, shared_dropout=0, loss_vel=None):
        super().__init__()
        if loss_iou is not None or iou_mlp is not None:
            _refuse("loss_iou / iou_mlp are not supported")
        if corner_loss_cfg is not None:
            _refuse("corner_loss_cfg is not supported")
        if enlarge_width is not None:
            _refuse("enlarge_width is not supported")
        if loss_vel is not None:
            _refuse("loss_vel is not supported")
        coder = dict(bbox_coder)
        if coder.get("type") != "BasePointBBoxCoder" or coder.get("code_size", 8) != 8:
            _refuse(f"bbox_coder must be BasePointBBoxCoder with code_size 8, got {coder}")
        _check_losses(loss_cls, dict(loss_center=loss_center, loss_size=loss_size, loss_rot=loss_rot))
        all_names = []
        for t in tasks:
            all_names += t['class_names']
        if all_names != list(class_names):
            _refuse(f"the tasks' class names {all_names} must equal class_names {list(class_names)}")
        self._build(num_classes, class_names, tasks, in_channel, shared_mlp_dims, norm_cfg, act, shared_dropout, common_attrs,
                    num_cls_layer, cls_hidden_dim, separate_head, train_cfg, test_cfg, as_rpn, loss_cls, loss_center, loss_size, loss_rot)

    def loss(self, cls_logits, reg_preds, cluster_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d, img_metas=None, iou_logits=None,
             gt_bboxes_ignore=None):
        """v2 lines 160-189: every task's loss_single_task in one targets launch and one fused loss; no host sync"""
        assert isinstance(cls_logits, list) and isinstance(reg_preds, list)
        assert len(cls_logits) == len(reg_preds) == len(self.tasks)
        return self._losses(list(range(len(self.tasks))), cls_logits, reg_preds, cluster_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d)

    def loss_single_task(self, task_id, cls_logits, reg_preds, cluster_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d, iou_logits=None):
        """v2 lines 192-297 for one task"""
        return self._losses([task_id], [cls_logits], [reg_preds], cluster_xyz, cluster_inds, gt_bboxes_3d, gt_labels_3d)

    def get_targets(self, num_task_classes, cluster_xyz, batch_idx, gt_bboxes_3d, gt_labels_3d, reg_preds=None):
        """v2 lines 328-347 for GTs whose labels are already within the task (modify_gt_for_single_task): (labels, label_weights,
        bbox_targets, bbox_weights, None) over the whole batch, from one launch"""
        return self._targets_one_task(num_task_classes, cluster_xyz, batch_idx, gt_bboxes_3d, gt_labels_3d)
