"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of Anchor3DHead's training path (mmdet3d/models/dense_heads/anchor3d_head.py, train_mixins.py) for the anchor-based SST
configs, pinned to the reference's own head by tests/test_oracle_anchor3d_vs_reference.py:

  anchors      AlignedAnchor3DRangeGenerator (anchor_3d_generator.py) in the reference's order ((y W + x) S + s) R + r
  targets      anchor_target_3d with one MaxIoUAssigner per size (mmdet 2.14 assign_wrt_overlaps) over the dense fp32 IoU matrix of
               BboxOverlapsNearest3D, PseudoSampler, DeltaXYZWLHRBBoxCoder.encode and get_direction_target
  losses       FocalLoss(use_sigmoid) / L1Loss with add_sin_difference / CrossEntropyLoss, in float64, differentiable
  get_bboxes   get_bboxes_single with rotated NMS (iou3d_oracle.box3d_multiclass_nms)

synth_batch / synth_preds make seeded batches with the edge cases the native kernels must get right."""
import math

import numpy as np
import torch

from oracle import iou3d_oracle as IO

PI4 = float(np.float32(np.pi / 4))
CLASS_SIZES = [[2.08, 4.73, 1.77], [0.84, 1.81, 1.77], [0.84, 0.91, 1.74]]   # car, cyclist, pedestrian (sst_base.py)
CLASS_Z = [-0.0345, -0.1188, 0.0]
CLASS_THR = [(0.55, 0.4, 0.4), (0.5, 0.3, 0.3), (0.5, 0.3, 0.3)]


def geometry(height=44, width=60, classes=(0, 1, 2), cell=0.64, rotations=(0, 1.57), assign_per_class=False, gt_max_assign_all=True,
             thresholds=None):
    """head kwargs (type popped) and train / test cfgs of a small SST-like Anchor3DHead: one anchor size per class in `classes`, an
    x / y range of width x height cells of `cell` metres centred on the origin"""
    hx, hy = width * cell / 2, height * cell / 2
    thr = thresholds or [CLASS_THR[c] for c in classes]
    gen = dict(type='AlignedAnchor3DRangeGenerator', ranges=[[-hx, -hy, CLASS_Z[c], hx, hy, CLASS_Z[c]] for c in classes],
               sizes=[CLASS_SIZES[c] for c in classes], rotations=list(rotations), reshape_out=False)
    assigner = [dict(type='MaxIoUAssigner', iou_calculator=dict(type='BboxOverlapsNearest3D'), pos_iou_thr=p, neg_iou_thr=n,
                     min_pos_iou=m, ignore_iof_thr=-1, gt_max_assign_all=gt_max_assign_all) for p, n, m in thr]
    train_cfg = dict(assigner=assigner, allowed_border=0, code_weight=[1.0] * 7, pos_weight=-1, debug=False)
    test_cfg = dict(use_rotate_nms=True, nms_across_levels=False, nms_pre=4096, nms_thr=0.25, score_thr=0.1, min_bbox_size=0, max_num=500)
    head = dict(num_classes=len(classes), in_channels=16, feat_channels=16, use_direction_classifier=True, anchor_generator=gen,
                assign_per_class=assign_per_class, diff_rad_by_sin=True, dir_offset=0.7854, dir_limit_offset=0,
                bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder', code_size=7),
                loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                loss_bbox=dict(type='L1Loss', loss_weight=0.5), loss_dir=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=0.2))
    return dict(head=head, train_cfg=train_cfg, test_cfg=test_cfg, H=height, W=width, S=len(classes), R=len(rotations))


def axes(geom):
    """(x_centers [W], y_centers [H], z [S], sizes [S, 3], rotations [R]) with anchors_single_range's fp32 arithmetic"""
    H, W = geom["H"], geom["W"]
    gen = geom["head"]["anchor_generator"]
    zs, whl = [], []
    for rng, size in zip(gen["ranges"], gen["sizes"]):
        r = torch.tensor(rng)
        z = torch.linspace(r[2], r[5], 2)
        y = torch.linspace(r[1], r[4], H + 1)
        x = torch.linspace(r[0], r[3], W + 1)
        z += (z[1] - z[0]) / 2
        y += (y[1] - y[0]) / 2
        x += (x[1] - x[0]) / 2
        zs.append(z[0])
        whl.append(torch.tensor(size).reshape(-1, 3)[0] * 1)
    return x[:W], y[:H], torch.stack(zs), torch.stack(whl), torch.tensor(gen["rotations"])


def anchors_from_axes(xc, yc, z, whl, rot):
    """[H, W, S, R, 7] anchors from the separable axes"""
    H, W, S, R = yc.numel(), xc.numel(), z.numel(), rot.numel()
    a = torch.empty((H, W, S, R, 7), dtype=torch.float32)
    a[..., 0] = xc.view(1, W, 1, 1)
    a[..., 1] = yc.view(H, 1, 1, 1)
    a[..., 2] = z.view(1, 1, S, 1)
    a[..., 3:6] = whl.view(1, 1, S, 1, 3)
    a[..., 6] = rot.view(1, 1, 1, R)
    return a


def limit_period(val, offset=0.5, period=np.pi):
    return val - torch.floor(val / period + offset) * period


def nearest_bev(boxes):
    """LiDARInstance3DBoxes.nearest_bev, fp32"""
    bev = boxes[:, [0, 1, 3, 4, 6]]
    normed = torch.abs(limit_period(bev[:, -1], 0.5, np.pi))
    xywh = torch.where((normed > np.pi / 4)[..., None], bev[:, [0, 1, 3, 2]], bev[:, :4])
    centers, dims = xywh[:, :2], xywh[:, 2:]
    return torch.cat([centers - dims / 2, centers + dims / 2], dim=-1)


def bbox_overlaps(b1, b2, eps=1e-6):
    """mmdet 2.14 bbox_overlaps, mode 'iou', not aligned"""
    if b1.shape[0] * b2.shape[0] == 0:
        return b1.new_zeros((b1.shape[0], b2.shape[0]))
    area1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    area2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt = torch.max(b1[..., :, None, :2], b2[..., None, :, :2])
    rb = torch.min(b1[..., :, None, 2:], b2[..., None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = area1[..., None] + area2[..., None, :] - overlap
    union = torch.max(union, union.new_tensor([eps]))
    return overlap / union


def assign(overlaps, pos_iou_thr, neg_iou_thr, min_pos_iou, gt_max_assign_all=True):
    """mmdet 2.14 MaxIoUAssigner.assign_wrt_overlaps (match_low_quality) -> assigned_gt_inds [A] (-1 ignored, 0 negative, i + 1)"""
    num_gts, num_bboxes = overlaps.shape
    assigned = overlaps.new_full((num_bboxes,), -1, dtype=torch.long)
    max_overlaps, argmax_overlaps = overlaps.max(dim=0)
    gt_max_overlaps, gt_argmax_overlaps = overlaps.max(dim=1)
    assigned[(max_overlaps >= 0) & (max_overlaps < neg_iou_thr)] = 0
    pos = max_overlaps >= pos_iou_thr
    assigned[pos] = argmax_overlaps[pos] + 1
    for i in range(num_gts):
        if gt_max_overlaps[i] >= min_pos_iou:
            if gt_max_assign_all:
                assigned[overlaps[i, :] == gt_max_overlaps[i]] = i + 1
            else:
                assigned[gt_argmax_overlaps[i]] = i + 1
    return assigned


def encode(src, dst):
    """DeltaXYZWLHRBBoxCoder.encode"""
    xa, ya, za, wa, la, ha, ra = torch.split(src, 1, dim=-1)
    xg, yg, zg, wg, lg, hg, rg = torch.split(dst, 1, dim=-1)
    za = za + ha / 2
    zg = zg + hg / 2
    diagonal = torch.sqrt(la**2 + wa**2)
    return torch.cat([(xg - xa) / diagonal, (yg - ya) / diagonal, (zg - za) / ha, torch.log(wg / wa), torch.log(lg / la),
                      torch.log(hg / ha), rg - ra], dim=-1)


def decode(anchors, deltas):
    """DeltaXYZWLHRBBoxCoder.decode"""
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, wt, lt, ht, rt = torch.split(deltas, 1, dim=-1)
    za = za + ha / 2
    diagonal = torch.sqrt(la**2 + wa**2)
    hg = torch.exp(ht) * ha
    zg = zt * ha + za - hg / 2
    return torch.cat([xt * diagonal + xa, yt * diagonal + ya, zg, torch.exp(wt) * wa, torch.exp(lt) * la, hg, rt + ra], dim=-1)


def direction_target(anchors, reg_targets, dir_offset):
    rot_gt = reg_targets[..., 6] + anchors[..., 6]
    offset_rot = limit_period(rot_gt - dir_offset, 0, 2 * np.pi)
    return torch.clamp(torch.floor(offset_rot / (2 * np.pi / 2)).long(), min=0, max=1)


def targets(anchors, gt_list, label_list, assigners, num_classes, assign_per_class=False, dir_offset=0.7854, ious=None, assigned=None):
    """anchor_target_3d restated.  anchors [H, W, S, R, 7]; gt_list / label_list: per sample [G, 7] bottom-centre / [G] int64;
    assigners: per size dicts (pos_iou_thr, neg_iou_thr, min_pos_iou, gt_max_assign_all).  Returns labels [B, A], label_weights,
    bbox_targets [B, A, 7], bbox_weights, dir_targets, dir_weights, num_total_pos (int).  `ious`, when a list, receives each (sample,
    size) IoU matrix; `assigned`, when a list, receives per sample the [A] sample-local index of each positive's GT (-1 elsewhere)."""
    H, W, S, R, _ = anchors.shape
    out = [[] for _ in range(6)]
    num_total_pos = 0
    for gt, lab in zip(gt_list, label_list):
        per = [[] for _ in range(6)]
        gidx = []
        npos = 0
        for s, asg in enumerate(assigners):
            anc = anchors[:, :, s].reshape(-1, 7)
            g, lb = (gt[lab == s], lab[lab == s]) if assign_per_class else (gt, lab)
            n = anc.shape[0]
            labels = torch.full((n,), num_classes, dtype=torch.long)
            lw = torch.zeros(n)
            bt, bw = torch.zeros(n, 7), torch.zeros(n, 7)
            dt, dw = torch.zeros(n, dtype=torch.long), torch.zeros(n)
            if g.shape[0] > 0:
                ov = bbox_overlaps(nearest_bev(g), nearest_bev(anc))
                if ious is not None:
                    ious.append(ov)
                gi = assign(ov, asg["pos_iou_thr"], asg["neg_iou_thr"], asg.get("min_pos_iou", 0.0), asg.get("gt_max_assign_all", True))
                pos, neg = torch.nonzero(gi > 0)[:, 0], torch.nonzero(gi == 0)[:, 0]
            else:
                pos, neg = torch.zeros(0, dtype=torch.long), torch.arange(n)
            gl = torch.full((n,), -1, dtype=torch.long)
            if pos.numel():
                gl[pos] = (torch.nonzero(lab == s)[:, 0] if assign_per_class else torch.arange(lab.numel()))[gi[pos] - 1]
            gidx.append(gl.reshape(H * W, 1, R))
            if pos.numel():
                t = encode(anc[pos], g[gi[pos] - 1])
                bt[pos], bw[pos] = t, 1.0
                dt[pos], dw[pos] = direction_target(anc[pos], t, dir_offset), 1.0
                labels[pos] = lb[gi[pos] - 1]
                lw[pos] = 1.0
            lw[neg] = 1.0
            npos += pos.numel()
            for k, v in enumerate((labels, lw, bt, bw, dt, dw)):
                per[k].append(v.reshape(H * W, 1, R, *v.shape[1:]))
        num_total_pos += max(npos, 1)
        if assigned is not None:
            assigned.append(torch.cat(gidx, 1).reshape(-1))
        for k in range(6):
            out[k].append(torch.cat(per[k], 1).reshape(H * W * S * R, *per[k][0].shape[3:]))
    return tuple(torch.stack(o) for o in out) + (num_total_pos,)


# ---- losses (float64, differentiable) ----
def focal_loss(cls_score, labels, label_weights, num_total_pos, num_classes, loss_weight=1.0, gamma=2.0, alpha=0.25):
    """mmdet 2.14 FocalLoss(use_sigmoid) py path on cls_score [B, A_loc C, H, W] permuted to [B A, C]"""
    x = cls_score.permute(0, 2, 3, 1).reshape(-1, num_classes)
    t = torch.nn.functional.one_hot(labels.reshape(-1), num_classes + 1)[:, :num_classes].to(x.dtype)
    p = x.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    fw = (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(x, t, reduction='none') * fw
    return loss_weight * (loss * label_weights.reshape(-1, 1).to(x.dtype)).sum() / num_total_pos


def reg_dir_loss(bbox_pred, dir_cls_preds, labels, bbox_targets, bbox_weights, dir_targets, dir_weights, num_total_pos, num_classes,
                 code_weight, w_bbox, w_dir):
    """loss_single's L1 (add_sin_difference) and direction cross-entropy over the positives"""
    labels = labels.reshape(-1)
    pos = torch.nonzero((labels >= 0) & (labels < num_classes))[:, 0]
    p = bbox_pred.permute(0, 2, 3, 1).reshape(-1, 7)[pos]
    d = dir_cls_preds.permute(0, 2, 3, 1).reshape(-1, 2)[pos]
    if pos.numel() == 0:
        return p.sum(), d.sum()
    t = bbox_targets.reshape(-1, 7)[pos]                # the targets' sin / cos in their own dtype, as add_sin_difference takes them
    w = bbox_weights.reshape(-1, 7)[pos] * bbox_weights.new_tensor(code_weight)
    p6 = torch.sin(p[:, 6:7]) * torch.cos(t[:, 6:7])
    t6 = torch.cos(p[:, 6:7]) * torch.sin(t[:, 6:7])
    p, t = torch.cat([p[:, :6], p6], 1), torch.cat([t[:, :6], t6], 1)
    lb = w_bbox * ((p - t).abs() * w).sum() / num_total_pos
    ce = torch.nn.functional.cross_entropy(d, dir_targets.reshape(-1)[pos], reduction='none')
    ld = w_dir * (ce * dir_weights.reshape(-1)[pos].to(d.dtype)).sum() / num_total_pos
    return lb, ld


# ---- decoding ----
def get_bboxes_single(cls_score, bbox_pred, dir_cls_pred, anchors, num_classes, test_cfg, dir_offset=0.7854, dir_limit_offset=0):
    """anchor3d_head.py get_bboxes_single for one level, rotated NMS; anchors [A, 7].  Returns (bboxes [N, 7], scores, labels)."""
    dir_score = torch.max(dir_cls_pred.permute(1, 2, 0).reshape(-1, 2), dim=-1)[1]
    scores = cls_score.permute(1, 2, 0).reshape(-1, num_classes).sigmoid()
    bbox_pred = bbox_pred.permute(1, 2, 0).reshape(-1, 7)
    nms_pre = test_cfg.get('nms_pre', -1)
    if nms_pre > 0 and scores.shape[0] > nms_pre:
        _, topk = scores.max(dim=1)[0].topk(nms_pre)
        anchors, bbox_pred, scores, dir_score = anchors[topk], bbox_pred[topk], scores[topk], dir_score[topk]
    bboxes = decode(anchors, bbox_pred)
    bev = bboxes[:, [0, 1, 3, 4, 6]]
    for_nms = torch.stack([bev[:, 0] - bev[:, 2] / 2, bev[:, 1] - bev[:, 3] / 2, bev[:, 0] + bev[:, 2] / 2, bev[:, 1] + bev[:, 3] / 2,
                           bev[:, 4]], 1)
    scores = torch.cat([scores, scores.new_zeros(scores.shape[0], 1)], 1)

    class Cfg(dict):
        __getattr__ = dict.__getitem__

    b, s, lab, d = IO.box3d_multiclass_nms(bboxes, for_nms, scores, test_cfg.get('score_thr', 0), test_cfg['max_num'], Cfg(test_cfg), dir_score)
    if b.shape[0] > 0:
        b[..., 6] = limit_period(b[..., 6] - dir_offset, dir_limit_offset, np.pi) + dir_offset + np.pi * d.to(b.dtype)
    return b, s, lab


# ---- synthetic data ----
def _f32(x):
    return float(np.float32(x))


def _ulp(x, k):
    """the fp32 k ulps away from fp32(x)"""
    v = np.float32(x)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
    return float(v)


def edge_yaws():
    """yaws at the nearest_bev swap boundary (|limit_period| = fp32 pi/4 and one ulp either side), at +-pi/2 and several periods out, and
    on the direction-bin boundaries (dir_offset 0.7854 + k pi) and one ulp either side"""
    ys = []
    for base in (PI4, -PI4, PI4 + math.pi, -PI4 - 3 * math.pi):
        ys += [_ulp(base, k) for k in (-1, 0, 1)]
    ys += [_f32(math.pi / 2), _f32(-math.pi / 2), _f32(math.pi / 2 + 4 * math.pi), _f32(-math.pi / 2 - 6 * math.pi)]
    for k in (-2, -1, 0, 1, 2):
        ys += [_ulp(0.7854 + k * math.pi, j) for j in (-1, 0, 1)]
    return ys


def synth_sample(seed, geom, n, edge=True):
    """[n, 7] bottom-centre GT boxes and int64 labels in a realistic class mix (60 % the first class) over the anchor range; with `edge`,
    boxes with the edge yaws, duplicates, boxes outside the range and zero-width boxes replace some of them"""
    g = torch.Generator().manual_seed(seed)
    S = geom["S"]
    gen = geom["head"]["anchor_generator"]
    hx, hy = gen["ranges"][0][3], gen["ranges"][0][4]
    if n == 0:
        return torch.zeros((0, 7)), torch.zeros((0,), dtype=torch.long)
    probs = torch.tensor([0.6] + [0.4 / max(S - 1, 1)] * (S - 1))[:S]
    lab = torch.multinomial(probs / probs.sum(), n, replacement=True, generator=g)
    size = torch.tensor(gen["sizes"])[lab] * (0.8 + 0.4 * torch.rand((n, 3), generator=g))
    ctr = (torch.rand((n, 2), generator=g) * 2 - 1) * torch.tensor([hx, hy]) * 0.95
    z = torch.tensor([r[2] for r in gen["ranges"]])[lab] + 0.2 * torch.randn(n, generator=g)
    yaw = (torch.rand(n, generator=g) * 2 - 1) * math.pi
    boxes = torch.cat([ctr, z[:, None], size, yaw[:, None]], 1).float()
    if edge and n >= 8:
        ys = edge_yaws()
        k = min(len(ys), n // 2)
        boxes[:k, 6] = torch.tensor(ys[:k])
        boxes[n // 2, :2] = torch.tensor([hx * 1.5, -hy * 1.3])          # outside the anchor range
        boxes[n // 2 + 1, 3] = 0.0                                         # zero width
        boxes[n - 1] = boxes[n - 2]                                        # duplicate GT
        lab[n - 1] = lab[n - 2]
        # a box centred on a cell centre, axis-aligned: many anchors of a size tie in IoU with it
        xc, yc, *_ = axes(geom)
        boxes[n - 3, :2] = torch.tensor([float(xc[len(xc) // 2]), float(yc[len(yc) // 2])])
        boxes[n - 3, 6] = 0.0
    return boxes.float(), lab.long()


def synth_batch(seed, geom, sizes, edge=True):
    out = [synth_sample(seed * 1000 + i, geom, n, edge) for i, n in enumerate(sizes)]
    return [b for b, _ in out], [lab for _, lab in out]


def synth_preds(seed, geom, batch, scale=1.0):
    """cls_score [B, S R C, H, W], bbox_pred [B, S R 7, H, W], dir_cls_preds [B, S R 2, H, W] fp32"""
    g = torch.Generator().manual_seed(seed)
    A_loc, C, H, W = geom["S"] * geom["R"], geom["head"]["num_classes"], geom["H"], geom["W"]
    cls = torch.randn((batch, A_loc * C, H, W), generator=g) * 2 * scale - 2
    reg = torch.randn((batch, A_loc * 7, H, W), generator=g) * 0.5 * scale
    dr = torch.randn((batch, A_loc * 2, H, W), generator=g) * scale
    return cls, reg, dr


def assigner_args(geom):
    return [dict(pos_iou_thr=a["pos_iou_thr"], neg_iou_thr=a["neg_iou_thr"], min_pos_iou=a.get("min_pos_iou", 0.0),
                 gt_max_assign_all=a.get("gt_max_assign_all", True)) for a in geom["train_cfg"]["assigner"]]
