"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of FSDV2Head's training and proposal paths (mmdet3d/models/dense_heads/fsd_v2_head.py) over
oracle/cluster_head_oracle.py's: the per-task targets with the in-box test on separate assignment points (centroid_assign) and the
velocity targets and weights of code size 10, the losses with loss_vel (mmdet's reduction 'mean' without avg_factor: over the
2 * num_pos elements) in whatever dtype the predictions have, and get_bboxes per (task, sample) then the all_task_max_num top-K.
Pinned to the reference's own head by tests/test_oracle_fsdv2_head_vs_reference.py; also the synthetic nuScenes-shaped clusters and
the config dicts the GPU tests and the benchmark use."""
import torch

from oracle import cluster_head_oracle as CO
from oracle import iou3d_oracle as IO
from oracle import roiaware_oracle as RA
from oracle import voteseg_oracle as VO

# configs/fsdv2/fsdv2_nusc_1x.py: 10 classes in two 5-class tasks
NUSC_NAMES = ['car', 'truck', 'trailer', 'bus', 'construction_vehicle', 'bicycle', 'motorcycle', 'pedestrian', 'traffic_cone', 'barrier']
NUSC_TASKS = [NUSC_NAMES[:5], NUSC_NAMES[5:]]

LOSS_MODES = {
    "nusc_l1": dict(gamma=2.0, alpha=0.25, loss_weight_cls=4.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                    smooth_l1=False, beta=1.0, loss_weight_vel=0.2),
    "nusc_smoothl1": dict(gamma=1.0, alpha=0.25, loss_weight_cls=4.0, loss_weight_center=0.5, loss_weight_size=0.5, loss_weight_rot=0.2,
                          smooth_l1=True, beta=0.1, loss_weight_vel=0.3),
}

# the `bbox_head` dict, train_cfg and test_cfg of configs/fsdv2/fsdv2_nusc_1x.py (pinned to the config by
# tests/test_oracle_fsdv2_head_vs_reference.py), for the GPU tests where the reference tree is absent
NUSC_HEAD = dict(
    type='FSDV2Head', num_classes=10, bbox_coder=dict(type='BasePointBBoxCoder', code_size=10),
    loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=4.0),
    loss_center=dict(type='L1Loss', loss_weight=0.5), loss_size=dict(type='L1Loss', loss_weight=0.5),
    loss_rot=dict(type='L1Loss', loss_weight=0.2), loss_vel=dict(type='L1Loss', loss_weight=0.2), in_channel=128,
    shared_mlp_dims=[256, 256], train_cfg=None, test_cfg=None, norm_cfg=dict(type='naiveSyncBN1d'),
    tasks=[dict(class_names=NUSC_TASKS[0]), dict(class_names=NUSC_TASKS[1])], class_names=NUSC_NAMES,
    common_attrs=dict(center=(3, 2, 128), dim=(3, 2, 128), rot=(2, 2, 128), vel=(2, 2, 128)), num_cls_layer=2, cls_hidden_dim=128,
    separate_head=dict(type='FSDSeparateHead', norm_cfg=dict(type='naiveSyncBN1d'), act='relu'))
_GROUPS = [['car'], ['truck', 'construction_vehicle'], ['bus', 'trailer'], ['barrier'], ['motorcycle', 'bicycle'],
           ['pedestrian', 'traffic_cone']]
NUSC_TRAIN_CFG = dict(score_thresh=[0.2] * 3 + [0.1] * 3, sync_reg_avg_factor=True, batched_group_sample=True, offset_weight='max',
                      class_names=NUSC_NAMES, group_names=_GROUPS, centroid_assign=True, disable_pretrain=True,
                      disable_pretrain_topks=[500] * 10)
NUSC_TEST_CFG = dict(score_thresh=[0.2] * 3 + [0.1] * 3, batched_group_sample=True, offset_weight='max', class_names=NUSC_NAMES,
                     group_names=_GROUPS, use_rotate_nms=True, nms_pre=-1, nms_thr=0.25, score_thr=0.05, min_bbox_size=0, max_num=500,
                     all_task_max_num=500)
# configs/fsdv2/fsdv2_waymo_1x.py: the head differs from FSD's D1 head in its MLP sizes and the training rpn cfg's nms_thr
WAYMO_HEAD = dict(CO.FSD_D1_HEAD, type='FSDV2Head', in_channel=128, shared_mlp_dims=[256, 256])
WAYMO_RPN_CFG = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=0.5, score_thr=0.1, min_bbox_size=0, max_num=500)
WAYMO_TRAIN_CFG = dict(score_thresh=(0.3, 0.25, 0.25), sync_reg_avg_factor=True, virtual_voxel_size=(0.5, 0.5, 0.5),
                       disable_pretrain=True, disable_pretrain_topks=[600, 200, 200], pre_2nd_voxelization=[0.1, 0.1, 0.1], rpn=WAYMO_RPN_CFG)


def encode(gt, xyz):
    """BasePointBBoxCoder.encode, code size 10 for 9 / 10-column boxes: the code-8 columns (log / sin / cos from float64, rounded
    once), then GT columns 7-8"""
    out = CO.encode(gt, xyz)
    return torch.cat([out, gt[:, 7:9].float()], 1) if gt.shape[1] >= 9 else out


def targets(xyz, bidx, boxes_list, labels_list, tasks, class_names, assign_xyz=None, code_size=8):
    """(labels, bbox_targets, num_pos): lists over tasks of int64 [M] and fp32 [M, 8] (code size 8) or [M, 11] (code size 10: the 10
    code columns and the velocity weight, the copy-paste flag of 10-column boxes or 1), and int64 [T].  The in-box test runs on
    assign_xyz when given, the encode on xyz."""
    M, B = xyz.shape[0], len(boxes_list)
    axyz = xyz if assign_xyz is None else assign_xyz
    cols = 11 if code_size == 10 else 8
    labels, tgs, nps = [], [], []
    for task in tasks:
        lab = torch.full((M,), len(task), dtype=torch.long)
        tg = torch.zeros((M, cols))
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
            gt = boxes_list[b][sel].float()
            hit = RA.points_in_boxes_gpu(axyz[rows, :3].float()[None], gt[None, :, :7])[0].long()
            pos = hit >= 0
            g = gt[hit[pos]]
            lab[rows[pos]] = rank[hit[pos]]
            if code_size == 10:
                w = g[:, 9:10] if g.shape[1] == 10 else torch.ones((g.shape[0], 1))
                tg[rows[pos]] = torch.cat([encode(g, xyz[rows[pos], :3].float()), w], 1)
            else:
                tg[rows[pos]] = CO.encode(g[:, :7], xyz[rows[pos], :3].float())
        bad = (bidx < 0) | (bidx >= B)
        lab[bad] = -1
        tg[bad] = float("nan")
        labels.append(lab)
        tgs.append(tg)
        nps.append(int(((lab >= 0) & (lab < len(task))).sum()))
    return labels, tgs, torch.tensor(nps, dtype=torch.long)


def losses(cls_logits, reg_preds, labels, bbox_targets, num_pos, cls_avg, reg_avg, gamma, alpha, loss_weight_cls, loss_weight_center,
           loss_weight_size, loss_weight_rot, smooth_l1, beta, loss_weight_vel=None):
    """[T, 4] = (cls, center, size, rot), or [T, 5] with vel when loss_weight_vel is given, per task in the predictions' dtype; vel is
    loss_weight_vel * sum(element * velocity weight) / (2 * num_pos), the regression 0 for a task without a local positive"""
    base = CO.losses(cls_logits, [r[:, :8] for r in reg_preds], labels, [t[:, :8] for t in bbox_targets], num_pos, cls_avg, reg_avg,
                     gamma, alpha, loss_weight_cls, loss_weight_center, loss_weight_size, loss_weight_rot, smooth_l1, beta)
    if loss_weight_vel is None:
        return base
    vel = []
    for t, (x, r, lab, tg) in enumerate(zip(cls_logits, reg_preds, labels, bbox_targets)):
        pos = (lab >= 0) & (lab < x.shape[1])
        n = int(num_pos[t])
        if n == 0:
            vel.append(r.sum() * 0)
            continue
        d = r[pos][:, 8:10] - tg[pos][:, 8:10].to(r.dtype)
        ad = d.abs()
        e = torch.where(ad < beta, 0.5 * ad * ad / beta, ad - 0.5 * beta) if smooth_l1 else ad
        vel.append(loss_weight_vel * (e * tg[pos][:, 10:11].to(r.dtype)).sum() / (2 * n))
    return torch.cat([base, torch.stack(vel)[:, None]], 1)


def decode(reg, base):
    out = CO.decode(reg[:, :8], base)
    return torch.cat([out, reg[:, 8:10]], 1) if reg.shape[1] == 10 else out


def get_bboxes(cls_logits, reg_preds, xyz, bidx, batch_size, tasks, class_names, cfg, all_task_max_num=None):
    """per sample (boxes [n, 7 | 9], scores, global labels) in the reference's order: per task, box3d_multiclass_nms of that sample's
    clusters on the CPU, the tasks concatenated, then a sample over all_task_max_num cut to its topk.  Given CUDA tensors, the decode
    and sigmoid run there first, so the boxes and scores are the reference's GPU results bit for bit"""
    cfg = CO.Cfg(cfg)
    out = []
    for b in range(batch_size):
        rows = bidx == b if batch_size > 1 else torch.ones_like(bidx, dtype=torch.bool)
        bb, ss, ll = [], [], []
        for t, task in enumerate(tasks):
            x, r, p = cls_logits[t][rows].float(), reg_preds[t][rows].float(), xyz[rows][:, :3].float()
            if x.shape[0] == 0:
                continue
            boxes = decode(r, p)
            scores = torch.cat([x.sigmoid(), x.new_zeros(x.shape[0], 1)], 1)
            boxes, scores, bfn = boxes.cpu(), scores.cpu(), CO.xywhr2xyxyr(boxes[:, [0, 1, 3, 4, 6]]).cpu()
            ob, os_, ol = IO.box3d_multiclass_nms(boxes, bfn, scores, cfg.get('score_thr', 0), cfg.max_num, cfg)[:3]
            glob = torch.tensor([class_names.index(n) for n in task], dtype=torch.long)
            bb.append(ob), ss.append(os_), ll.append(glob[ol] if ol.numel() else ol.long())
        dim = 9 if reg_preds[0].shape[1] == 10 else 7
        res = (torch.cat(bb) if bb else torch.zeros((0, dim)), torch.cat(ss) if ss else torch.zeros((0,)),
               torch.cat(ll) if ll else torch.zeros((0,), dtype=torch.long))
        if all_task_max_num is not None and res[1].shape[0] > all_task_max_num:
            k = res[1].topk(all_task_max_num)[1]
            res = tuple(a[k] for a in res)
        out.append(res)
    return out


# ---- synthetic data ----
def synth_clusters(seed, n_clusters, n_boxes, class_names=NUSC_NAMES, width=9, paste=0.3, spread=30.0, inside=0.6, voxel=0.4):
    """cluster_xyz [M, 3] (voxel centres), their point centroids [M, 3] (within half a voxel of the centre), cluster_inds int64 [M, 3]
    with samples interleaved, and per sample boxes [G_b, width] (bottom-centre, velocities in columns 7-8, for width 10 a copy-paste
    flag in column 9 that is 0 for about `paste` of them) and global labels.  Boxes overlap in pairs across classes."""
    g = torch.Generator().manual_seed(seed)
    K = len(class_names)
    cen, bi, Bx, Lb = [], [], [], []
    for b, (n, m) in enumerate(zip(n_clusters, n_boxes)):
        boxes, _ = VO.synth_boxes(g, m, 3, spread, 0.0)
        if m > 1:
            boxes[1::2] = boxes[0:-1:2]
        vel = torch.randn((m, 2), generator=g) * 3
        extra = [vel]
        if width == 10:
            extra.append((torch.rand((m, 1), generator=g) >= paste).float())
        boxes = torch.cat([boxes] + extra, 1)
        lab = torch.randint(0, K, (m,), generator=g)
        pts = VO.points_around(g, boxes[:, :7], n, spread, cols=3, inside=inside)
        cen.append(pts)
        bi.append(torch.full((n,), b, dtype=torch.long))
        Bx.append(boxes)
        Lb.append(lab)
    cen, bi = torch.cat(cen), torch.cat(bi)
    o = torch.randperm(cen.shape[0], generator=g)
    cen, bi = cen[o], bi[o]
    xyz = cen + (torch.rand(cen.shape, generator=g) - 0.5) * voxel     # the voxel centre, off the centroid by under half a voxel
    inds = torch.stack([torch.randint(0, K, bi.shape, generator=g), bi, torch.arange(bi.shape[0])], 1)
    return xyz.contiguous(), cen.contiguous(), inds, Bx, Lb


def synth_preds(seed, M, tasks, code_size=10, scale=3.0):
    """cls_logits [M, C_t] and reg_preds [M, code_size] per task, fp32"""
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn((M, len(t)), generator=g) * scale for t in tasks], [torch.randn((M, code_size), generator=g) for t in tasks])
