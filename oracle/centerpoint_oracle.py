"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CenterHead's training path restated on the CPU (mmdet3d/models/dense_heads/centerpoint_head.py:421-610):
  targets   the reference's fp32 op sequence of get_targets_single in torch, vectorised over boxes (every op is the same correctly
            rounded elementwise fp32 op as on the reference's 0-d tensors), drawn with the numpy gaussian_2d of
            mmdet3d/core/utils/gaussian.py:5-57;
  losses    in float64, after mmdet 2.14.0 (docs/overall_instructions.md:20; mmdet is not in the tree, so these are unpinned externals):
            models/losses/gaussian_focal_loss.py (alpha 2, gamma 4, eps 1e-12), smooth_l1_loss.py L1Loss, and utils.py
            weight_reduce_loss (reduction 'mean' with avg_factor: loss.sum() / avg_factor, no eps in 2.14);
  decode    CenterPointBBoxCoder.decode (core/bbox/coders/centerpoint_bbox_coders.py) and CenterHead.get_task_detections with
            oracle/iou3d_oracle.py's NMS.
Also the synthetic cases the tests share: the two geometries and the semantic edge cases."""
import math

import numpy as np
import torch

from oracle import iou3d_oracle as IO

# configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py:84-140
WAYMO = dict(tasks=[3], train_cfg=dict(grid_size=[468, 468, 1], voxel_size=(0.32, 0.32, 6), out_size_factor=1, dense_reg=1,
                                       gaussian_overlap=0.1, max_objs=500, min_radius=2,
                                       point_cloud_range=[-74.88, -74.88, -2, 74.88, 74.88, 4],
                                       code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0, 0.0]),
             box_dim=7, loss_bbox_weight=2.0,
             bbox_coder=dict(type='CenterPointBBoxCoder', post_center_range=[-74.88, -74.88, -10.0, 74.88, 74.88, 10.0], max_num=4096,
                             score_threshold=0.1, out_size_factor=1, voxel_size=(0.32, 0.32), pc_range=[-74.88, -74.88], code_size=9),
             test_cfg=dict(post_center_limit_range=[-80, -80, -10, 80, 80, 10], max_per_img=500, max_pool_nms=False,
                           min_radius=[4, 12, 10, 1, 0.85, 0.175], score_threshold=0.1, pc_range=[-74.88, -74.88], out_size_factor=1,
                           voxel_size=(0.32, 0.32), nms_type='rotate', pre_max_size=4096, post_max_size=500, nms_thr=0.7))
# tests/test_models/test_heads/test_heads.py:768-850 (the reference's own unit test of the DCN CenterHead)
NUSC = dict(tasks=[1, 2, 2, 1, 2, 2], train_cfg=dict(grid_size=[512, 512, 1], point_cloud_range=[-51.2, -51.2, -5., 51.2, 51.2, 3.],
                                                   voxel_size=[0.2, 0.2, 8], out_size_factor=4, dense_reg=1, gaussian_overlap=0.1,
                                                   max_objs=500, min_radius=2,
                                                   code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2, 1.0, 1.0]),
            box_dim=9, loss_bbox_weight=0.25,
            bbox_coder=dict(type='CenterPointBBoxCoder', post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], max_num=500,
                            score_threshold=0.1, pc_range=[-51.2, -51.2], out_size_factor=4, voxel_size=[0.2, 0.2], code_size=9),
            test_cfg=dict(post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], max_per_img=500, max_pool_nms=False,
                          min_radius=[4, 12, 10, 1, 0.85, 0.175], post_max_size=83, score_threshold=0.1, pc_range=[-51.2, -51.2],
                          out_size_factor=4, voxel_size=[0.2, 0.2], nms_type='rotate', pre_max_size=1000, nms_thr=0.2))
GEOMETRIES = {"waymo": WAYMO, "nusc": NUSC}


def geometry(width, height, out_size_factor=1, voxel_size=(0.32, 0.32), gaussian_overlap=0.1, min_radius=2, max_objs=500, tasks=(3,),
             box_dim=7):
    """a GEOMETRIES-style dict for a width x height feature map (grid_size = map * out_size_factor), the point-cloud range centred on
    the origin; the rest as WAYMO, with the code weights of NUSC (none zero)"""
    vx, vy = voxel_size
    gx, gy = width * out_size_factor, height * out_size_factor
    pc = [-0.5 * gx * vx, -0.5 * gy * vy, -2.0, 0.5 * gx * vx, 0.5 * gy * vy, 4.0]
    return dict(tasks=list(tasks), box_dim=box_dim, loss_bbox_weight=2.0,
                train_cfg=dict(grid_size=[gx, gy, 1], voxel_size=(vx, vy, 6), out_size_factor=out_size_factor, dense_reg=1,
                               gaussian_overlap=gaussian_overlap, max_objs=max_objs, min_radius=min_radius, point_cloud_range=pc,
                               code_weights=list(NUSC['train_cfg']['code_weights'])),
                bbox_coder=dict(type='CenterPointBBoxCoder', post_center_range=[pc[0] - 10, pc[1] - 10, -10.0, pc[3] + 10, pc[4] + 10, 10.0],
                                max_num=500, score_threshold=0.1, out_size_factor=out_size_factor, voxel_size=(vx, vy), pc_range=pc[:2],
                                code_size=9),
                test_cfg=dict(post_center_limit_range=[pc[0] - 10, pc[1] - 10, -10.0, pc[3] + 10, pc[4] + 10, 10.0], max_per_img=500,
                              max_pool_nms=False, min_radius=[4, 12, 10, 1, 0.85, 0.175], post_max_size=83, score_threshold=0.1,
                              pc_range=pc[:2], out_size_factor=out_size_factor, voxel_size=(vx, vy), nms_type='rotate', pre_max_size=1000,
                              nms_thr=0.2))


def _geom(geom):
    return GEOMETRIES[geom] if isinstance(geom, str) else geom


def head_cfg(geom, in_channels=16, share_conv_channel=8, dcn=False):
    """a CenterHead config dict of GEOMETRIES[geom] or of a geometry() dict (the regression heads of both CenterHead configs;
    SeparateHead unless dcn)"""
    G = _geom(geom)
    names = [[f"c{i}_{j}" for j in range(n)] for i, n in enumerate(G['tasks'])]
    sep = dict(type='SeparateHead', init_bias=-2.19, final_kernel=3)
    if dcn:
        sep = dict(type='DCNSeparateHead', init_bias=-2.19, final_kernel=3,
                   dcn_config=dict(type='DCN', in_channels=share_conv_channel, out_channels=share_conv_channel, kernel_size=3, padding=1,
                                   groups=4, bias=False))
    return dict(type='CenterHead', in_channels=in_channels, tasks=[dict(num_class=len(n), class_names=n) for n in names],
                common_heads=dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)), share_conv_channel=share_conv_channel,
                bbox_coder=dict(G['bbox_coder']), separate_head=sep, loss_cls=dict(type='GaussianFocalLoss', reduction='mean'),
                loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=G['loss_bbox_weight']), norm_bbox=True,
                train_cfg=dict(G['train_cfg']), test_cfg=dict(G['test_cfg']))


def feature_map_size(cfg):
    osf = cfg['out_size_factor']
    return cfg['grid_size'][0] // osf, cfg['grid_size'][1] // osf


def gaussian_2d(shape, sigma=1):
    """mmdet3d/core/utils/gaussian.py:5-21"""
    m, n = [(ss - 1.) / 2. for ss in shape]
    y, x = np.ogrid[-m:m + 1, -n:n + 1]
    h = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    h[h < np.finfo(h.dtype).eps * h.max()] = 0
    return h


def _draw(heatmap, x, y, radius):
    """draw_heatmap_gaussian (gaussian.py:24-57), k = 1, on a [H, W] fp32 tensor"""
    diameter = 2 * radius + 1
    gaussian = gaussian_2d((diameter, diameter), sigma=diameter / 6)
    height, width = heatmap.shape[0:2]
    left, right = min(x, radius), min(width - x, radius + 1)
    top, bottom = min(y, radius), min(height - y, radius + 1)
    masked_heatmap = heatmap[y - top:y + bottom, x - left:x + right]
    masked_gaussian = torch.from_numpy(gaussian[radius - top:radius + bottom, radius - left:radius + right]).to(torch.float32)
    if min(masked_gaussian.shape) > 0 and min(masked_heatmap.shape) > 0:
        torch.max(masked_heatmap, masked_gaussian, out=masked_heatmap)


def gaussian_radius(height, width, min_overlap):
    """gaussian.py:60-87 on fp32 tensors, elementwise; Python's min(r1, r2, r3) as two strict comparisons"""
    a1 = 1
    b1 = (height + width)
    c1 = width * height * (1 - min_overlap) / (1 + min_overlap)
    sq1 = torch.sqrt(b1**2 - 4 * a1 * c1)
    r1 = (b1 + sq1) / 2
    a2 = 4
    b2 = 2 * (height + width)
    c2 = (1 - min_overlap) * width * height
    sq2 = torch.sqrt(b2**2 - 4 * a2 * c2)
    r2 = (b2 + sq2) / 2
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    c3 = (min_overlap - 1) * width * height
    sq3 = torch.sqrt(b3**2 - 4 * a3 * c3)
    r3 = (b3 + sq3) / 2
    r = torch.where(r2 < r1, r2, r1)
    return torch.where(r3 < r, r3, r)


def targets_single(boxes, labels, task_num_classes, cfg, norm_bbox=True):
    """get_targets_single for one sample: boxes [N, 7|9] fp32 with a gravity-centre z, labels int64 [N] -> per task (heatmap
    [ncls, H, W], anno_box [max_objs, 10], ind [max_objs], mask [max_objs])"""
    max_objs = cfg['max_objs'] * cfg['dense_reg']
    pc_range = torch.tensor(cfg['point_cloud_range'])
    voxel_size = torch.tensor(cfg['voxel_size'])
    osf = cfg['out_size_factor']
    W, H = feature_map_size(cfg)
    out, flag = [], 0
    for ncls in task_num_classes:
        order = torch.cat([torch.where(labels == flag + c)[0] for c in range(ncls)])[:max_objs]
        cls = labels[order] - flag
        flag += ncls
        b = boxes[order]
        heatmap = torch.zeros((ncls, H, W), dtype=torch.float32)
        anno_box = torch.zeros((max_objs, 10), dtype=torch.float32)
        ind = torch.zeros((max_objs,), dtype=torch.int64)
        mask = torch.zeros((max_objs,), dtype=torch.uint8)
        width = b[:, 3] / voxel_size[0] / osf
        length = b[:, 4] / voxel_size[1] / osf
        radius = gaussian_radius(length, width, cfg['gaussian_overlap'])
        coor_x = (b[:, 0] - pc_range[0]) / voxel_size[0] / osf
        coor_y = (b[:, 1] - pc_range[1]) / voxel_size[1] / osf
        center = torch.stack([coor_x, coor_y], 1)
        center_int = center.to(torch.int32)
        ok = (width > 0) & (length > 0) & (center_int[:, 0] >= 0) & (center_int[:, 0] < W) & (center_int[:, 1] >= 0) & \
             (center_int[:, 1] < H)
        for k in torch.nonzero(ok)[:, 0].tolist():
            r = max(cfg['min_radius'], int(radius[k]))
            _draw(heatmap[int(cls[k])], int(center_int[k, 0]), int(center_int[k, 1]), r)
        ind[:b.shape[0]][ok] = center_int[ok, 1].long() * W + center_int[ok, 0].long()
        mask[:b.shape[0]][ok] = 1
        box_dim = b[:, 3:6].log() if norm_bbox else b[:, 3:6]
        vel = b[:, 7:9] if b.shape[1] >= 9 else torch.zeros((b.shape[0], 2), dtype=torch.float32)
        rows = torch.cat([center - center_int.float(), b[:, 2:3], box_dim, torch.sin(b[:, 6:7]), torch.cos(b[:, 6:7]), vel], 1)
        anno_box[:b.shape[0]][ok] = rows[ok]
        out.append((heatmap, anno_box, ind, mask))
    return out


def targets(boxes_list, labels_list, task_num_classes, cfg, norm_bbox=True):
    """get_targets: four lists over tasks of [B, ...] tensors"""
    per = [targets_single(b, l, task_num_classes, cfg, norm_bbox) for b, l in zip(boxes_list, labels_list)]
    return tuple([torch.stack([p[t][i] for p in per]) for t in range(len(task_num_classes))] for i in range(4))


def gravity(boxes):
    """LiDARInstance3DBoxes.gravity_center in fp32 (lidar_box3d.py:45-51) concatenated with the rest of the box"""
    return torch.cat([boxes[:, :2], boxes[:, 2:3] + boxes[:, 5:6] * 0.5, boxes[:, 3:]], 1)


# ---- losses (float64) ----
def clip_sigmoid(x, eps=1e-4):
    return torch.clamp(x.sigmoid(), min=eps, max=1 - eps)


def gaussian_focal_loss(pred, gaussian_target, alpha=2.0, gamma=4.0):
    """mmdet 2.14 models/losses/gaussian_focal_loss.py, elementwise"""
    eps = 1e-12
    pos_weights = gaussian_target.eq(1)
    neg_weights = (1 - gaussian_target).pow(gamma)
    pos_loss = -(pred + eps).log() * (1 - pred).pow(alpha) * pos_weights
    neg_loss = -(1 - pred + eps).log() * pred.pow(alpha) * neg_weights
    return pos_loss + neg_loss


def focal_loss(logits, target, loss_weight=1.0):
    """GaussianFocalLoss(reduction='mean') of CenterHead.loss on clip_sigmoid(logits), avg_factor max(num_pos, 1) -> (loss, num_pos)"""
    num_pos = float(target.eq(1).sum())
    return loss_weight * gaussian_focal_loss(clip_sigmoid(logits), target).sum() / max(num_pos, 1), num_pos


def l1_loss(preds, anno_box, ind, mask, code_weights, loss_weight):
    """CenterHead.loss's regression term: L1Loss(reduction='mean') with weight mask * notnan * code_weights, avg_factor sum(mask) + 1e-4
    (in fp32, as the reference computes it)"""
    pred = torch.cat([preds['reg'], preds['height'], preds['dim'], preds['rot'], preds['vel']], 1)
    pred = pred.permute(0, 2, 3, 1).reshape(pred.shape[0], -1, pred.shape[1])
    pred = pred.gather(1, ind.unsqueeze(2).expand(ind.shape[0], ind.shape[1], pred.shape[2]))
    target = anno_box.to(pred.dtype)
    m = mask.unsqueeze(2).expand_as(target).to(pred.dtype) * (~torch.isnan(target)).to(pred.dtype)
    w = m * torch.tensor(code_weights, dtype=torch.float32).to(pred.dtype)     # fp32 code weights, as mask.new_tensor() makes them
    avg_factor = (mask.float().sum() + 1e-4).to(pred.dtype)        # the reference forms it in fp32 from masks.float()
    return loss_weight * ((pred - target).abs() * w).sum() / avg_factor


# ---- decode ----
def _gather(feats, inds):
    return feats.gather(1, inds.unsqueeze(2).expand(inds.size(0), inds.size(1), feats.size(2)))


def _tg(feat, ind):
    feat = feat.permute(0, 2, 3, 1).contiguous()
    return _gather(feat.view(feat.size(0), -1, feat.size(3)), ind)


def decode(heat, rot_sine, rot_cosine, hei, dim, vel, reg, coder):
    """CenterPointBBoxCoder.decode -> [dict(bboxes, scores, labels)] per sample"""
    batch, cat, height, width = heat.size()
    K = coder['max_num']
    topk_scores, topk_inds = torch.topk(heat.view(batch, cat, -1), K)
    topk_inds = topk_inds % (height * width)
    ys = (topk_inds.float() / torch.tensor(width, dtype=torch.float)).int().float()
    xs = (topk_inds % width).int().float()
    scores, topk_ind = torch.topk(topk_scores.view(batch, -1), K)
    clses = (topk_ind / torch.tensor(K, dtype=torch.float)).int()
    inds = _gather(topk_inds.view(batch, -1, 1), topk_ind).view(batch, K)
    ys = _gather(ys.view(batch, -1, 1), topk_ind).view(batch, K, 1)
    xs = _gather(xs.view(batch, -1, 1), topk_ind).view(batch, K, 1)
    reg = _tg(reg, inds).view(batch, K, 2)
    xs, ys = xs + reg[:, :, 0:1], ys + reg[:, :, 1:2]
    rot = torch.atan2(_tg(rot_sine, inds).view(batch, K, 1), _tg(rot_cosine, inds).view(batch, K, 1))
    hei = _tg(hei, inds).view(batch, K, 1)
    dim = _tg(dim, inds).view(batch, K, 3)
    xs = xs * coder['out_size_factor'] * coder['voxel_size'][0] + coder['pc_range'][0]
    ys = ys * coder['out_size_factor'] * coder['voxel_size'][1] + coder['pc_range'][1]
    boxes = torch.cat([xs, ys, hei, dim, rot, _tg(vel, inds).view(batch, K, 2)], 2)
    pcr = torch.tensor(coder['post_center_range'])
    mask = (boxes[..., :3] >= pcr[:3]).all(2) & (boxes[..., :3] <= pcr[3:]).all(2)
    if coder['score_threshold']:
        mask &= scores > coder['score_threshold']
    return [dict(bboxes=boxes[i, mask[i]], scores=scores[i, mask[i]], labels=clses[i, mask[i]].float()) for i in range(batch)]


def bev_xyxyr(boxes):
    """xywhr2xyxyr of the LiDAR BEV columns (0, 1, 3, 4, 6)"""
    b = boxes[:, [0, 1, 3, 4, 6]]
    hw, hh = b[:, 2] / 2, b[:, 3] / 2
    return torch.stack([b[:, 0] - hw, b[:, 1] - hh, b[:, 0] + hw, b[:, 1] + hh, b[:, 4]], 1)


def get_bboxes(preds_dicts, num_classes, coder, test_cfg, norm_bbox=True):
    """CenterHead.get_bboxes with rotated NMS -> [[bboxes [N, 9] bottom-centre z, scores, labels int32]] per sample"""
    rets = []
    for task_id, pd in enumerate(preds_dicts):
        p = pd[0]
        temp = decode(p['heatmap'].sigmoid(), p['rot'][:, 0:1], p['rot'][:, 1:2], p['height'],
                      torch.exp(p['dim']) if norm_bbox else p['dim'], p['vel'], p['reg'], coder)
        task = []
        pcr = torch.tensor(test_cfg['post_center_limit_range'], dtype=torch.float32)
        for t in temp:
            boxes, scores = t['bboxes'], t['scores']
            labels = torch.zeros(scores.shape[0], dtype=torch.long) if num_classes[task_id] == 1 else t['labels'].long()
            if test_cfg['score_threshold'] > 0.0:
                keep = scores >= test_cfg['score_threshold']
                boxes, scores, labels = boxes[keep], scores[keep], labels[keep]
            sel = IO.nms_gpu(bev_xyxyr(boxes), scores, test_cfg['nms_thr'], test_cfg['pre_max_size'], test_cfg['post_max_size']) \
                if scores.shape[0] else torch.zeros((0,), dtype=torch.long)
            boxes, scores, labels = boxes[sel], scores[sel], labels[sel]
            m = (boxes[:, :3] >= pcr[:3]).all(1) & (boxes[:, :3] <= pcr[3:]).all(1)
            task.append((boxes[m], scores[m], labels[m]))
        rets.append(task)
    out = []
    for i in range(len(rets[0])):
        boxes = torch.cat([r[i][0] for r in rets])
        boxes[:, 2] = boxes[:, 2] - boxes[:, 5] * 0.5
        flag, labels = 0, []
        for j, n in enumerate(num_classes):
            labels.append((rets[j][i][2] + flag).int())
            flag += n
        out.append([boxes, torch.cat([r[i][1] for r in rets]), torch.cat(labels)])
    return out


# ---- synthetic cases ----
def synth_sample(seed, cfg, n, ncls_total, box_dim, edge=True):
    """one sample's raw LiDAR boxes [n (+ edge cases), box_dim] (bottom-centre z) and int64 labels.  Edge cases: centres at the map's
    corners and edges, in (-1, 0) cells and outside the map, zero and negative sizes, duplicate centre cells, a box larger than the map,
    labels outside every task, and sizes bisected to put the fp32 radius within an ulp of an integer."""
    g = torch.Generator().manual_seed(seed)
    pc, vs, osf = cfg['point_cloud_range'], cfg['voxel_size'], cfg['out_size_factor']
    W, H = feature_map_size(cfg)
    cell_x, cell_y = vs[0] * osf, vs[1] * osf
    xy = torch.rand(n, 2, generator=g, dtype=torch.float64)
    x = pc[0] + xy[:, 0] * (pc[3] - pc[0])
    y = pc[1] + xy[:, 1] * (pc[4] - pc[1])
    dims = torch.rand(n, 3, generator=g, dtype=torch.float64) * torch.tensor([4.0, 9.0, 3.0], dtype=torch.float64) + 0.3
    rows = [torch.stack([x, y, -1 + torch.rand(n, generator=g, dtype=torch.float64)], 1), dims,
            (torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1) * math.pi]
    if box_dim == 9:
        rows.append(torch.randn(n, 2, generator=g, dtype=torch.float64) * 3)
    boxes = torch.cat(rows, 1).float()
    labels = torch.randint(0, ncls_total, (n,), generator=g)
    if edge:
        ex = []
        corners = [(0.01, 0.01), (W - 0.01, 0.01), (0.01, H - 0.01), (W - 0.01, H - 0.01), (W / 2, 0.3), (0.3, H / 2), (W - 0.3, H / 2),
                   (-0.5, 3.3), (3.3, -0.7), (-1.5, 4.0), (W + 0.5, 2.0), (2.0, H + 0.2), (7.5, 7.5), (7.6, 7.4), (7.5, 7.5)]
        for cx, cy in corners:   # map cells -> metres
            ex.append([pc[0] + cx * cell_x, pc[1] + cy * cell_y, 0.0, 2.0, 4.5, 1.6, 0.3])
        ex += [[pc[0] + 20.5 * cell_x, pc[1] + 30.5 * cell_y, 0.0, 0.0, 4.0, 1.5, 0.1],     # zero width
               [pc[0] + 21.5 * cell_x, pc[1] + 31.5 * cell_y, 0.0, 2.0, -1.0, 1.5, 0.1],    # negative length
               [pc[0] + 40.5 * cell_x, pc[1] + 41.5 * cell_y, 0.0, 3.0 * W * cell_x, 3.0 * H * cell_y, 2.0, 0.0]]  # radius beyond the map
        ex += [[pc[0] + (50.5 + 3 * k) * cell_x, pc[1] + 60.5 * cell_y, 0.0, w, l, 1.5, 0.2] for k, (w, l) in
               enumerate(near_integer_sizes(cfg, 4))]
        ex = torch.tensor(ex, dtype=torch.float32)
        if box_dim == 9:
            ex = torch.cat([ex, torch.randn(ex.shape[0], 2, generator=g)], 1)
        ex_labels = torch.randint(0, ncls_total, (ex.shape[0],), generator=g)
        ex_labels[-5] = ncls_total + 3                    # a label outside every task
        boxes, labels = torch.cat([boxes, ex]), torch.cat([labels, ex_labels])
        perm = torch.randperm(boxes.shape[0], generator=g)
        boxes, labels = boxes[perm], labels[perm]
    return boxes, labels


def near_integer_sizes(cfg, count):
    """(dx, dy) metre pairs whose fp32 gaussian_radius lies within an ulp of an integer (found by bisection on dx)"""
    vs, osf, o = cfg['voxel_size'], cfg['out_size_factor'], cfg['gaussian_overlap']
    out = []
    for target in range(3, 3 + count):
        lo, hi = 0.05, 40.0
        dy = 2.5 * vs[1] * osf * target
        length = torch.tensor([dy], dtype=torch.float32) / torch.tensor(vs)[1] / osf
        f = lambda dx: float(gaussian_radius(length, torch.tensor([dx], dtype=torch.float32) / torch.tensor(vs)[0] / osf, o)[0])
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if f(mid) < target else (lo, mid)
        out.append((float(np.float32(lo)), dy))
        out.append((float(np.float32(hi)), dy))
    return out[:count]


def synth_batch(seed, geom, sizes, edge=True):
    """raw boxes / labels per sample for GEOMETRIES[geom] or a geometry() dict; sizes: boxes per sample (0 = an empty sample)"""
    G = _geom(geom)
    ncls = sum(G['tasks'])
    out = [synth_sample(seed * 97 + i, G['train_cfg'], n, ncls, G['box_dim'], edge=edge and n > 0) for i, n in enumerate(sizes)]
    return [o[0] for o in out], [o[1] for o in out]


def synth_preds(seed, geom, batch, scale=1.0):
    """random head outputs (heatmap logits per task and the five regression heads) for GEOMETRIES[geom] or a geometry() dict, fp32"""
    G = _geom(geom)
    W, H = feature_map_size(G['train_cfg'])
    g = torch.Generator().manual_seed(seed)
    out = []
    for ncls in G['tasks']:
        p = {k: torch.randn(batch, c, H, W, generator=g) * scale for k, c in (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))}
        p['heatmap'] = torch.randn(batch, ncls, H, W, generator=g) * 3 - 2
        out.append([p])
    return out
