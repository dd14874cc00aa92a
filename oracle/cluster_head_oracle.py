"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of SparseClusterHeadV2's training and proposal paths (mmdet3d/models/dense_heads/sparse_cluster_head{,_v2}.py):
get_targets per task after modify_gt_for_single_task (the first in-box hit over the task's GTs ordered by class rank, then input index),
BasePointBBoxCoder.encode with its log / sin / cos in float64 rounded once, the per-task losses of loss_single_task in whatever dtype the
predictions have (float64 for the gradient checks, through autograd), and get_bboxes per (task, sample) over oracle/iou3d_oracle.py's
box3d_multiclass_nms.  Pinned to the reference's own head by tests/test_oracle_cluster_head_vs_reference.py; also the synthetic
clusters the GPU tests and the benchmark use."""
import math

import torch
import torch.nn.functional as F

from oracle import iou3d_oracle as IO
from oracle import roiaware_oracle as RA
from oracle import voteseg_oracle as VO

WAYMO_NAMES = ['Car', 'Pedestrian', 'Cyclist']
WAYMO_TASKS = [['Car'], ['Pedestrian'], ['Cyclist']]
# configs/argo2/argo_onestage_12e.py: 26 classes in six multi-class groups
ARGO_NAMES = [f"a{i}" for i in range(26)]
ARGO_TASKS = [ARGO_NAMES[0:4], ARGO_NAMES[4:9], ARGO_NAMES[9:13], ARGO_NAMES[13:18], ARGO_NAMES[18:22], ARGO_NAMES[22:26]]

LOSS_MODES = {
    "fsd_l1": dict(gamma=2.0, alpha=0.25, loss_weight_cls=2.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                   smooth_l1=False, beta=1.0),
    "argo_smoothl1": dict(gamma=1.0, alpha=0.25, loss_weight_cls=1.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                          smooth_l1=True, beta=0.1),
    "fsd_smoothl1": dict(gamma=2.0, alpha=0.25, loss_weight_cls=2.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                         smooth_l1=True, beta=0.1),
    "argo_l1": dict(gamma=1.0, alpha=0.25, loss_weight_cls=1.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                    smooth_l1=False, beta=1.0),
}

RPN_CFG = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=None, score_thr=0.1, min_bbox_size=0, max_num=500)
TEST_CFG = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=0.25, score_thr=0.1, min_bbox_size=0, max_num=500)


class Cfg(dict):
    """mmcv ConfigDict's attribute access"""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError:
            raise AttributeError(k)
        return Cfg(v) if isinstance(v, dict) else v


def encode(gt, xyz):
    """BasePointBBoxCoder.encode in fp32, its log / sin / cos in float64 rounded once"""
    delta = gt[:, :3] - xyz
    log_dims = (gt[:, 3:6] + 1e-6).double().log().float()
    yaw = gt[:, 6:7].double()
    return torch.cat([delta, log_dims, yaw.sin().float(), yaw.cos().float()], 1)


def targets(xyz, bidx, boxes_list, labels_list, tasks, class_names):
    """(labels, bbox_targets, num_pos): lists over tasks of int64 [M] and fp32 [M, 8], and int64 [T]"""
    M, B = xyz.shape[0], len(boxes_list)
    labels, tgs, nps = [], [], []
    for task in tasks:
        lab = torch.full((M,), len(task), dtype=torch.long)
        tg = torch.zeros((M, 8))
        for b in range(B):
            rows = torch.nonzero(bidx == b)[:, 0]
            sel, rank = [], []
            for r, n in enumerate(task):
                k = torch.nonzero(labels_list[b] == class_names.index(n))[:, 0]
                sel.append(k)
                rank.append(torch.full_like(k, r))
            sel, rank = torch.cat(sel), torch.cat(rank)
            if rows.numel() == 0 or sel.numel() == 0:
                continue
            gt = boxes_list[b][sel][:, :7].float()
            p = xyz[rows, :3].float()
            hit = RA.points_in_boxes_gpu(p[None], gt[None])[0].long()
            pos = hit >= 0
            lab[rows[pos]] = rank[hit[pos]]
            tg[rows[pos]] = encode(gt[hit[pos]], p[pos])
        bad = (bidx < 0) | (bidx >= B)
        lab[bad] = -1
        tg[bad] = float("nan")
        labels.append(lab)
        tgs.append(tg)
        nps.append(int(((lab >= 0) & (lab < len(task))).sum()))
    return labels, tgs, torch.tensor(nps, dtype=torch.long)


def losses(cls_logits, reg_preds, labels, bbox_targets, num_pos, cls_avg, reg_avg, gamma, alpha, loss_weight_cls, loss_weight_center,
           loss_weight_size, loss_weight_rot, smooth_l1, beta):
    """[T, 4] = (cls, center, size, rot) per task in the predictions' dtype; regression 0 for a task without a local positive"""
    out = []
    for t, (x, r, lab, tg) in enumerate(zip(cls_logits, reg_preds, labels, bbox_targets)):
        C = x.shape[1]
        onehot = F.one_hot(lab.clamp(min=0), C + 1)[:, :C].to(x.dtype)
        p = x.sigmoid()
        fl = alpha * onehot * (1 - p).pow(gamma) * F.softplus(-x) + (1 - alpha) * (1 - onehot) * p.pow(gamma) * F.softplus(x)
        cls = fl.sum()
        if (lab < 0).any():
            cls = cls + float("nan")
        row = [loss_weight_cls * cls / float(cls_avg[t])]
        pos = (lab >= 0) & (lab < C)
        d = r[pos] - tg[pos].to(r.dtype)
        ad = d.abs()
        e = torch.where(ad < beta, 0.5 * ad * ad / beta, ad - 0.5 * beta) if smooth_l1 else ad
        for w, (a, b) in zip((loss_weight_center, loss_weight_size, loss_weight_rot), ((0, 3), (3, 6), (6, 8))):
            row.append(w * e[:, a:b].sum() / float(reg_avg[t]) if int(num_pos[t]) > 0 else r.sum() * 0)
        out.append(torch.stack(row))
    return torch.stack(out)


def xywhr2xyxyr(b):
    out = torch.zeros_like(b)
    hw, hh = b[:, 2] / 2, b[:, 3] / 2
    out[:, 0], out[:, 1], out[:, 2], out[:, 3], out[:, 4] = b[:, 0] - hw, b[:, 1] - hh, b[:, 0] + hw, b[:, 1] + hh, b[:, 4]
    return out


def decode(reg, base):
    return torch.cat([reg[:, :3] + base, reg[:, 3:6].exp() - 1e-6, torch.atan2(reg[:, 6:7], reg[:, 7:8])], 1)


def get_bboxes(cls_logits, reg_preds, xyz, bidx, batch_size, tasks, class_names, cfg):
    """per sample (boxes [n, 7], scores, global labels) in the reference's order: per task, box3d_multiclass_nms of that sample's
    clusters, on the CPU.  Given CUDA tensors, the decode, sigmoid and xywhr2xyxyr run there first, so the boxes and scores are the
    reference's GPU results bit for bit"""
    cfg = Cfg(cfg)
    out = []
    for b in range(batch_size):
        rows = bidx == b if batch_size > 1 else torch.ones_like(bidx, dtype=torch.bool)   # split_by_batch: every row for a batch of one
        bb, ss, ll = [], [], []
        for t, task in enumerate(tasks):
            x, r, p = cls_logits[t][rows].float(), reg_preds[t][rows].float(), xyz[rows][:, :3].float()
            if x.shape[0] == 0:
                continue
            boxes = decode(r, p)
            scores = torch.cat([x.sigmoid(), x.new_zeros(x.shape[0], 1)], 1)
            boxes, scores, bfn = boxes.cpu(), scores.cpu(), xywhr2xyxyr(boxes[:, [0, 1, 3, 4, 6]]).cpu()
            ob, os_, ol = IO.box3d_multiclass_nms(boxes, bfn, scores, cfg.get('score_thr', 0), cfg.max_num, cfg)[:3]
            glob = torch.tensor([class_names.index(n) for n in task], dtype=torch.long)
            bb.append(ob), ss.append(os_), ll.append(glob[ol] if ol.numel() else ol.long())
        out.append((torch.cat(bb) if bb else torch.zeros((0, 7)), torch.cat(ss) if ss else torch.zeros((0,)),
                    torch.cat(ll) if ll else torch.zeros((0,), dtype=torch.long)))
    return out


# ---- synthetic data ----
def synth_clusters(seed, n_clusters, n_boxes, class_names=WAYMO_NAMES, spread=40.0, invalid=0.0, shuffle=True, inside=0.6):
    """cluster_xyz [M, 3], cluster_inds int64 [M, 3] (class, sample, cluster id; samples interleaved when shuffle), and the boxes /
    global labels per sample; boxes overlap in pairs across classes, some yaws are +-pi"""
    g = torch.Generator().manual_seed(seed)
    K = len(class_names)
    xyz, bi, Bx, Lb = [], [], [], []
    for b, (n, m) in enumerate(zip(n_clusters, n_boxes)):
        boxes, _ = VO.synth_boxes(g, m, 3, spread, 0.0)
        lab = torch.randint(0, K, (m,), generator=g)
        if m:
            lab[torch.rand(m, generator=g) < invalid] = -1
        pts = VO.points_around(g, boxes, n, spread, cols=3, inside=inside)
        xyz.append(pts)
        bi.append(torch.full((n,), b, dtype=torch.long))
        Bx.append(boxes)
        Lb.append(lab)
    xyz, bi = torch.cat(xyz), torch.cat(bi)
    if shuffle:
        o = torch.randperm(xyz.shape[0], generator=g)
        xyz, bi = xyz[o], bi[o]
    inds = torch.stack([torch.randint(0, K, bi.shape, generator=g), bi, torch.arange(bi.shape[0])], 1)
    return xyz.contiguous(), inds, Bx, Lb


def synth_preds(seed, M, tasks, scale=3.0):
    """cls_logits [M, C_t] and reg_preds [M, 8] per task, fp32"""
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn((M, len(t)), generator=g) * scale for t in tasks], [torch.randn((M, 8), generator=g) for t in tasks])


def yaw_pi(boxes):
    boxes[::3, 6] = torch.tensor([math.pi, -math.pi], dtype=torch.float32).repeat(boxes.shape[0])[:boxes[::3].shape[0]]
    return boxes


# the `bbox_head` dict of configs/fsd/fsd_waymoD1_1x.py and its train / test rpn cfgs (pinned to the config by
# tests/test_oracle_cluster_head_vs_reference.py), for the GPU tests where the reference tree is absent
FSD_D1_HEAD = dict(
    type='SparseClusterHeadV2', num_classes=3, bbox_coder=dict(type='BasePointBBoxCoder'),
    loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=2.0),
    loss_center=dict(type='L1Loss', loss_weight=0.5), loss_size=dict(type='L1Loss', loss_weight=0.5),
    loss_rot=dict(type='L1Loss', loss_weight=0.2), in_channel=128 * 3 * 2, shared_mlp_dims=[1024, 1024], train_cfg=None, test_cfg=None,
    norm_cfg=dict(type='LN'), tasks=[dict(class_names=['Car']), dict(class_names=['Pedestrian']), dict(class_names=['Cyclist'])],
    class_names=WAYMO_NAMES, common_attrs=dict(center=(3, 2, 128), dim=(3, 2, 128), rot=(2, 2, 128)), num_cls_layer=2, cls_hidden_dim=128,
    separate_head=dict(type='FSDSeparateHead', norm_cfg=dict(type='LN'), act='relu'), as_rpn=True)
FSD_D1_TRAIN_CFG = dict(score_thresh=(0.3, 0.25, 0.25), sync_reg_avg_factor=True, pre_voxelization_size=(0.1, 0.1, 0.1),
                        disable_pretrain=True, disable_pretrain_topks=[600, 200, 200], rpn=RPN_CFG)
FSD_D1_TEST_CFG = dict(score_thresh=(0.3, 0.25, 0.25), pre_voxelization_size=(0.1, 0.1, 0.1), rpn=TEST_CFG)
