"""CPU restatement of FSD's second stage in float64: GroupCorrectionHead._assign_and_sample (fsd_roi_head.py:213-296, mmdet 2.14
MaxIoUAssigner.assign_wrt_overlaps, IoUNegPiecewiseSampler), FullySparseBboxHead._get_target_single, loss and get_bboxes
(fsd_bbox_head.py).  random_choice(gallery, k) keeps the k gallery members with the smallest keys (ties to the lower proposal index),
the rule the native sampler follows.  Boxes are LiDAR bottom-centre (x, y, z, w, l, h, yaw[, vx, vy])."""
import math

import numpy as np
import torch

from oracle import iou3d_oracle as IO


def xyxyr(b):
    b = b.double()
    return torch.stack([b[:, 0] - b[:, 3] / 2, b[:, 1] - b[:, 4] / 2, b[:, 0] + b[:, 3] / 2, b[:, 1] + b[:, 4] / 2, b[:, 6]], 1)


def iou3d(gt, props):
    """LiDARInstance3DBoxes.overlaps(gt, props) in float64: [G, N]"""
    if len(gt) == 0 or len(props) == 0:
        return torch.zeros((len(gt), len(props)), dtype=torch.float64)
    g, p = gt.double(), props.double()
    ov = IO.boxes_overlap_bev(xyxyr(g), xyxyr(p))
    h = (torch.min((g[:, 2] + g[:, 5])[:, None], (p[:, 2] + p[:, 5])[None]) - torch.max(g[:, 2][:, None], p[:, 2][None])).clamp(min=0)
    ov3 = ov * h
    v = lambda b: b[:, 3] * b[:, 4] * b[:, 5]  # noqa: E731
    return ov3 / (v(g)[:, None] + v(p)[None] - ov3).clamp(min=1e-8)


def assign(overlaps, gt_labels, pos, neg, min_pos):
    """assign_wrt_overlaps with match_low_quality and gt_max_assign_all: (gt_inds 1-based / 0 / -1, max_overlaps, labels)"""
    G, N = overlaps.shape
    gi = torch.full((N,), -1, dtype=torch.int64)
    if G == 0 or N == 0:
        if G == 0:
            gi[:] = 0
        return gi, torch.zeros(N, dtype=torch.float64), torch.full((N,), -1, dtype=torch.int64)
    mo, arg = overlaps.max(0)
    gmax = overlaps.max(1)[0]
    gi[(mo >= 0) & (mo < neg)] = 0
    p = mo >= pos
    gi[p] = arg[p] + 1
    for i in range(G):
        if gmax[i] >= min_pos:
            gi[overlaps[i] == gmax[i]] = i + 1
    lab = torch.full((N,), -1, dtype=torch.int64)
    lab[gi > 0] = gt_labels[gi[gi > 0] - 1]
    return gi, mo, lab


def choose(gallery, k, keys):
    """random_choice(gallery, k) under the key rule: the k members with the smallest (key, index)"""
    order = sorted(range(len(gallery)), key=lambda t: (float(keys[gallery[t]]), int(gallery[t])))
    return gallery[torch.tensor(order[:k], dtype=torch.int64)]


def sample(gi, mo, keys, num, pos_fraction, fractions, thrs):
    """IoUNegPiecewiseSampler.sample with neg_pos_ub < 0 and no GT proposals -> (pos_inds, neg_inds), each ascending"""
    pos = torch.nonzero(gi > 0).view(-1)
    npe = int(num * pos_fraction)
    if len(pos) > npe:
        pos = choose(pos, npe, keys)
    pos = pos.unique()
    nexp = num - len(pos)
    neg = torch.nonzero(gi == 0).view(-1)
    if len(neg) > nexp:
        choice, extend = neg.new_zeros([0]), 0
        m = mo[neg]
        for q in range(len(fractions)):
            if q == len(fractions) - 1:
                want, lo = nexp - len(choice), 0
            else:
                want, lo = int(nexp * fractions[q]) + extend, thrs[q + 1]
            piece = neg[(m >= lo) & (m < thrs[q])]
            if len(piece) < want:
                choice = torch.cat([choice, piece])
                extend += want - len(piece)
            else:
                choice = torch.cat([choice, choose(piece, want, keys)])
                extend = 0
        neg = choice
    return pos, neg.unique()


def assign_and_sample(props, plabels, keys, gt, gl, assigners, per_class, num, pos_fraction, fractions, thrs):
    """one sample -> (inds, iou, gt_rows (sample-local, -1 on negatives), labels, num_pos); assigners: (pos, neg, min_pos) per class"""
    N = len(props)
    gi = torch.zeros(N, dtype=torch.int64)
    mo = torch.zeros(N, dtype=torch.float64)
    lab = torch.full((N,), -1, dtype=torch.int64)
    if per_class:
        for i, (p, n, m) in enumerate(assigners):
            gm, pm = gl == i, plabels == i
            g_i, mo_i, l_i = assign(iou3d(gt[gm], props[pm]), gl[gm], p, n, m)
            pad = torch.cat([torch.tensor([-1, 0]), torch.nonzero(gm).view(-1) + 1])
            gi[pm], mo[pm], lab[pm] = pad[g_i + 1], mo_i, l_i
    else:
        gi, mo, lab = assign(iou3d(gt, props), gl, *assigners[0])
    pos, neg = sample(gi, mo, keys, num, pos_fraction, fractions, thrs)
    inds = torch.cat([pos, neg])
    rows = torch.cat([gi[pos] - 1, torch.full((len(neg),), -1, dtype=torch.int64)])
    return inds, mo[inds], rows, torch.cat([lab[pos], torch.full((len(neg),), -1, dtype=torch.int64)]), len(pos)


def rot(xyz, a):
    s, c = torch.sin(a), torch.cos(a)
    return torch.stack([xyz[:, 0] * c + xyz[:, 1] * s, -xyz[:, 0] * s + xyz[:, 1] * c, xyz[:, 2]], 1)


def targets(rois, iou, gt, labels, pos_thr, neg_thr):
    """_get_target_single on positive rows (gt, labels) and every row's soft label: (soft [R], bbox_targets [Npos, 7])"""
    R, npos = len(iou), len(gt)
    soft = torch.zeros(R, dtype=torch.float64)
    for r in range(npos):
        c, v = int(labels[r]), float(iou[r])
        soft[r] = 1.0 if v > pos_thr[c] else (0.0 if v < neg_thr[c] else (v - neg_thr[c]) / (pos_thr[c] - neg_thr[c]))
    p, g = rois[:npos, :7].double(), gt[:, :7].double()
    ry = torch.remainder(p[:, 6], 2 * math.pi)
    ct = g.clone()
    ct[:, :3] = rot(g[:, :3] - p[:, :3], -(ry + math.pi / 2))
    yl = torch.remainder(g[:, 6] - ry, 2 * math.pi)
    opp = (yl > math.pi / 2) & (yl < math.pi * 1.5)
    yl[opp] = torch.remainder(yl[opp] + math.pi, 2 * math.pi)
    yl[yl > math.pi] -= 2 * math.pi
    yl = yl.clamp(-math.pi / 2, math.pi / 2)
    diag = torch.sqrt(p[:, 4] ** 2 + p[:, 3] ** 2)
    bt = torch.stack([ct[:, 0] / diag, ct[:, 1] / diag, (ct[:, 2] + ct[:, 5] / 2 - p[:, 5] / 2) / p[:, 5], torch.log(g[:, 3] / p[:, 3]),
                      torch.log(g[:, 4] / p[:, 4]), torch.log(g[:, 5] / p[:, 5]), yl], 1)
    return soft, bt


def corners(b):
    u = torch.tensor([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]], dtype=b.dtype)
    u = u - u.new_tensor([0.5, 0.5, 0])
    c = b[:, None, 3:6] * u[None]
    s, co = torch.sin(b[:, 6])[:, None], torch.cos(b[:, 6])[:, None]
    c = torch.stack([c[..., 0] * co + c[..., 1] * s, -c[..., 0] * s + c[..., 1] * co, c[..., 2]], -1)
    return c + b[:, None, :3]


def decode(rois, pred):
    """the loss' decode: DeltaXYZWLHR against the RoI with xyz = 0, rotated by roi yaw + pi / 2, shifted to the RoI"""
    a = rois[:, :7]
    ha, wa, la = a[:, 5], a[:, 3], a[:, 4]
    diag = torch.sqrt(la ** 2 + wa ** 2)
    h = torch.exp(pred[:, 5]) * ha
    loc = torch.stack([pred[:, 0] * diag, pred[:, 1] * diag, pred[:, 2] * ha + ha / 2 - h / 2], 1)
    xyz = rot(loc, a[:, 6] + math.pi / 2) + a[:, :3]
    return torch.cat([xyz, (torch.exp(pred[:, 3]) * wa)[:, None], (torch.exp(pred[:, 4]) * la)[:, None], h[:, None],
                      (pred[:, 6] + a[:, 6])[:, None]], 1)


def losses(cls_score, bbox_pred, nonempty, soft, reg_mask, bbox_targets_rows, pos_gt_rows, labels_rows, rois, cfg):
    """FullySparseBboxHead.loss in float64 (torch autograd gives the gradient): dict of the three losses.  The *_rows tensors are
    row-aligned with the RoIs.  cfg: w_cls, w_bbox, smooth_l1, beta, code_weights, with_corner, corner_class, w_corner, cls_avg,
    reg_avg (None: the positive count)"""
    x = cls_score.view(-1)
    y = soft.double()
    w = nonempty.double()
    bce = torch.clamp(x, min=0) - x * y + torch.log1p(torch.exp(-x.abs()))
    out = {'loss_rcnn_cls': cfg['w_cls'] * (bce * w).sum() / cfg.get('cls_avg', float(len(x)))}
    pos = (reg_mask > 0) & nonempty
    n = int(pos.sum())
    if n == 0:
        out['loss_rcnn_bbox'] = bbox_pred.sum() * 0
        out['loss_rcnn_corner'] = bbox_pred.sum() * 0
        return out
    d = bbox_pred[pos] - bbox_targets_rows[pos].double()
    if cfg['smooth_l1']:
        e = torch.where(d.abs() < cfg['beta'], 0.5 * d * d / cfg['beta'], d.abs() - 0.5 * cfg['beta'])
    else:
        e = d.abs()
    cw = torch.tensor(cfg.get('code_weights') or [1.0] * 7, dtype=torch.float64)
    out['loss_rcnn_bbox'] = cfg['w_bbox'] * (e * cw).sum() / (cfg.get('reg_avg') or n)
    sel = pos & (labels_rows == cfg['corner_class']) if cfg['corner_class'] >= 0 else pos
    if not cfg['with_corner'] or int(sel.sum()) == 0:
        out['loss_rcnn_corner'] = bbox_pred.sum() * 0
        return out
    pb = decode(rois[sel].double(), bbox_pred[sel])
    g = pos_gt_rows[sel].double()
    gf = g.clone()
    gf[:, 6] += math.pi
    pc, gc, fc = corners(pb), corners(g), corners(gf)
    dist = torch.min(torch.norm(pc - gc, dim=2), torch.norm(pc - fc, dim=2))
    q = dist.clamp(max=1.0)
    out['loss_rcnn_corner'] = cfg['w_corner'] * (0.5 * q ** 2 + (dist - q)).mean()
    return out


def decode_from_rois(rois, bbox_pred):
    rb = rois[:, 1:].double()
    local = rb.clone()
    local[:, :3] = 0
    pred = bbox_pred.double()
    if rb.shape[1] == 9:
        pred = torch.cat([pred, pred.new_zeros((len(pred), 2))], 1)
    a = local
    diag = torch.sqrt(a[:, 4] ** 2 + a[:, 3] ** 2)
    h = torch.exp(pred[:, 5]) * a[:, 5]
    loc = torch.stack([pred[:, 0] * diag, pred[:, 1] * diag, pred[:, 2] * a[:, 5] + a[:, 5] / 2 - h / 2], 1)
    out = [rot(loc, rb[:, 6] + math.pi / 2) + rb[:, :3], (torch.exp(pred[:, 3]) * a[:, 3])[:, None],
           (torch.exp(pred[:, 4]) * a[:, 4])[:, None], h[:, None], (pred[:, 6] + a[:, 6])[:, None]]
    if rb.shape[1] == 9:
        out.append(pred[:, 7:9] + a[:, 7:9])
    return torch.cat(out, 1)


def get_bboxes(rois, cls_score, bbox_pred, valid, labels, probs, num_classes, score_thr, nms_thr, rcnn_score_nms=False):
    """get_bboxes + multi_class_nms (rotated) for a batch of one -> (boxes, scores, labels)"""
    s = torch.sigmoid(cls_score.double()).view(-1)
    if rcnn_score_nms:
        probs = s.clone()
    rois, s, bbox_pred, labels, probs = rois[valid], s[valid], bbox_pred[valid], labels[valid], probs[valid].double()
    boxes = decode_from_rois(rois, bbox_pred)
    sel = []
    for k in range(num_classes):
        m = (probs >= score_thr) & (labels == k)
        if m.any():
            idx = torch.nonzero(m).view(-1)
            keep = IO.nms_gpu(xyxyr(boxes[idx]).float(), probs[idx].float(), nms_thr)
            sel.append(idx[keep])
    sel = torch.cat(sel) if sel else torch.zeros(0, dtype=torch.int64)
    return boxes[sel], s[sel], labels[sel]


# ---- synthetic inputs ------------------------------------------------------------------------------------------------------------
def synth_sample(seed, n_props, n_gt, num_classes=3, spread=40.0, width=7, gt_width=7):
    """proposals jittered around GTs (and some far ones), with predicted labels mostly the GT's: (props, plabels, gt, gl)"""
    g = torch.Generator().manual_seed(seed)
    size = torch.tensor([[2.0, 4.5, 1.6], [0.8, 0.8, 1.8], [0.8, 1.8, 1.6]])
    gl = torch.randint(0, num_classes, (n_gt,), generator=g)
    gt = torch.zeros((n_gt, gt_width))
    gt[:, :2] = (torch.rand(n_gt, 2, generator=g) * 2 - 1) * spread
    gt[:, 2] = torch.rand(n_gt, generator=g) - 1
    gt[:, 3:6] = size[gl % 3] * (1 + 0.1 * torch.randn(n_gt, 3, generator=g)).clamp(0.7, 1.3)
    gt[:, 6] = (torch.rand(n_gt, generator=g) * 2 - 1) * math.pi
    if gt_width > 7:
        gt[:, 7:9] = torch.randn(n_gt, 2, generator=g)
    if gt_width > 9:
        gt[:, 9] = 1.0
    props = torch.zeros((n_props, width))
    if n_gt:
        k = torch.randint(0, n_gt, (n_props,), generator=g)
        props[:, :7] = gt[k, :7]
        props[:, :3] += torch.randn(n_props, 3, generator=g) * torch.tensor([0.6, 0.6, 0.2])
        props[:, 3:6] *= (1 + 0.15 * torch.randn(n_props, 3, generator=g)).clamp(0.6, 1.4)
        props[:, 6] += 0.3 * torch.randn(n_props, generator=g)
        far = torch.rand(n_props, generator=g) < 0.2
        props[far, :2] = (torch.rand(int(far.sum()), 2, generator=g) * 2 - 1) * spread
        plab = torch.where(torch.rand(n_props, generator=g) < 0.85, gl[k], torch.randint(0, num_classes, (n_props,), generator=g))
    else:
        props[:, :2] = (torch.rand(n_props, 2, generator=g) * 2 - 1) * spread
        props[:, 3:6] = size[0]
        plab = torch.randint(0, num_classes, (n_props,), generator=g)
    return props, plab, gt, gl


def near_threshold(props, plab, gt, gl, thrs, per_class=True, margin=1e-4):
    """True when any (proposal, GT) IoU the assigner sees lies within margin of one of thrs"""
    ov = iou3d(gt, props)
    if per_class:
        ov = torch.where(gl[:, None] == plab[None], ov, torch.full_like(ov, -1.0))
    return any(bool(((ov - t).abs() < margin).any()) for t in thrs)
