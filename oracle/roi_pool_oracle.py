"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of FSD's RoI point pooling (SURVEY 8f next-3): dynamic_point_pool / dynamic_point_pool_mixed
(mmdet3d/ops/dynamic_point_pool_op.py:9-113) as DynamicPointROIExtractor uses them
(mmdet3d/models/roi_heads/roi_extractors/dynamic_point_roi_extractor.py:32-136).  Dense: every box against every point, then a stable
selection.  Pinned: tests/test_oracle_roi_pool_vs_reference.py runs the box test against the reference's own points_in_boxes_cpu,
compiled unmodified into oracle/_ref by oracle/build_ref_roiaware.py."""
import math

import torch


def box_test(pts, boxes):
    """check_pt_in_box3d (mmdet3d/ops/roiaware_pool3d/src/points_in_boxes_cuda.cu:24-49, CPU twin points_in_boxes_cpu.cpp:16-40) for every
    (box, point): inside [R, N] bool, local x / y [R, N] fp32, box centre z [R].  The fp32 steps of the CUDA kernel: centre z = bottom +
    h / 2 in double, angle rz + pi / 2 in double then fp32, cos / sin of that fp32 angle (correctly rounded here), and the contraction nvcc
    applies to `sx * cos + sy * (-sin)` / `sx * sin + sy * cos`: the product with cos is fused, the one with sin rounded first."""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    cx, cy, zb, w, l, h, rz = boxes.unbind(1)
    cz = (zb.double() + h.double() / 2).float()
    ang = (rz.double() + math.pi / 2).float().double()
    ca, sa = torch.cos(ang).float(), torch.sin(ang).float()
    sx, sy = x[None] - cx[:, None], y[None] - cy[:, None]
    lx = (sx.double() * ca.double()[:, None] - (sy * sa[:, None]).double()).float()
    ly = (sy.double() * ca.double()[:, None] + (sx * sa[:, None]).double()).float()
    inside = ~((z[None] - cz[:, None]).abs() > (h / 2)[:, None])
    inside &= (lx > -(l / 2)[:, None]) & (lx < (l / 2)[:, None]) & (ly > -(w / 2)[:, None]) & (ly < (w / 2)[:, None])
    return inside, lx, ly, cz


def enlarge_boxes(boxes, extra_wlh):
    """same centre and yaw, dims (w + e0, l + e1, h + e2): (x, y, z_bottom - e2 / 2, w + e0, l + e1, h + e2, rz), fp32"""
    cx, cy, zb, w, l, h, rz = boxes.unbind(1)
    e0, e1, e2 = (float(v) for v in extra_wlh)
    return torch.stack([cx, cy, zb - 0.5 * e2, w + e0, l + e1, h + e2, rz], 1)


def dynamic_point_pool(rois, pts, extra_wlh, max_inbox_point, max_all_pts=50000, rois_batch=None, pts_batch=None, chunk=32):
    """Dense restatement of the op's contract (the kernel itself, TorchEx dynamic_point_pool_ext, is not in the reference tree):
      pinned by the reference: box layout (x, y, z_bottom, w, l, h, rz) (dynamic_point_roi_extractor.py:63,117), the in-box test above,
      feature layout [xyz, local_xyz, 6 boundary offsets, is_in_margin] (:87-90), offset identities off[0]+off[3] = l, off[1]+off[4] = w,
      off[2]+off[5] = h and out_xyz == pts[idx] (:92-101), one fake row (-1, -1, zeros) when nothing pairs (dynamic_point_pool_op.py:36-46);
      chosen here (include/sstb200.h): a pair = point inside the enlarged box; is_in_margin = inside the enlarged box but not the original;
      local_xyz = (local x, local y, z - centre z); offsets against the original box; rows sorted by RoI then point index, every RoI keeps
      its first max_inbox_point points; max_all_pts caps the call in (RoI, point) order; mixed: pairs need equal batch ids."""
    rois, pts = rois.float(), pts[:, :3].float()
    big = enlarge_boxes(rois, extra_wlh)
    idx_l, roi_l, feat_l = [], [], []
    for r0 in range(0, rois.shape[0], chunk):
        sl = slice(r0, r0 + chunk)
        in_e, lx, ly, _ = box_test(pts, big[sl])
        in_o, _, _, cz = box_test(pts, rois[sl])
        if rois_batch is not None:
            in_e &= rois_batch[sl].long()[:, None] == pts_batch.long()[None]
        for j in range(in_e.shape[0]):
            r = r0 + j
            idx = in_e[j].nonzero()[:, 0][:max_inbox_point]
            if idx.numel() == 0:
                continue
            p = pts[idx]
            loc = torch.stack([lx[j, idx], ly[j, idx], p[:, 2] - cz[j]], 1)
            half = torch.stack([rois[r, 4], rois[r, 3], rois[r, 5]]) / 2
            feat_l.append(torch.cat([p, loc, half + loc, half - loc, (~in_o[j, idx]).float()[:, None]], 1))
            idx_l.append(idx)
            roi_l.append(torch.full_like(idx, r))
    if not idx_l:
        return torch.full((1,), -1, dtype=torch.long), torch.full((1,), -1, dtype=torch.long), torch.zeros((1, 13))
    return torch.cat(idx_l)[:max_all_pts], torch.cat(roi_l)[:max_all_pts], torch.cat(feat_l)[:max_all_pts]


def synth_roi_frame(seed, n_pts=100000, n_rois=500, spread=60.0, batch_size=1):
    """an FSD-shaped second-stage input: points concentrated around objects plus background, RoIs of car / pedestrian / cyclist size
    (w, l, h) with random yaw placed on most objects; returns pts [N, 3], rois [R, 7] (x, y, z_bottom, w, l, h, rz), batch ids of both"""
    g = torch.Generator().manual_seed(seed)
    sizes = torch.tensor([[2.0, 4.5, 1.6], [0.8, 0.9, 1.8], [0.8, 1.8, 1.7]])
    cls = torch.randint(0, 3, (n_rois,), generator=g)
    wlh = sizes[cls] * (0.8 + 0.4 * torch.rand((n_rois, 3), generator=g))
    xy = (torch.rand((n_rois, 2), generator=g) - 0.5) * 2 * spread
    zb = -1.8 + 0.3 * torch.randn((n_rois, 1), generator=g)
    rz = (torch.rand((n_rois, 1), generator=g) - 0.5) * 2 * math.pi
    rois = torch.cat([xy, zb, wlh, rz], 1)
    n_obj = n_pts // 2
    pick = torch.randint(0, n_rois, (n_obj,), generator=g)
    obj = torch.cat([xy[pick], zb[pick] + wlh[pick, 2:3] / 2], 1) + torch.randn((n_obj, 3), generator=g) * torch.cat(
        [wlh[pick, 1:2] / 2, wlh[pick, 1:2] / 2, wlh[pick, 2:3] / 3], 1)
    bg = torch.cat([(torch.rand((n_pts - n_obj, 2), generator=g) - 0.5) * 2 * (spread + 10), torch.rand((n_pts - n_obj, 1), generator=g) * 4 - 2.5], 1)
    pts = torch.cat([obj, bg])[torch.randperm(n_pts, generator=g)]
    rb = torch.sort(torch.randint(0, batch_size, (n_rois,), generator=g))[0].int()
    pb = torch.sort(torch.randint(0, batch_size, (n_pts,), generator=g))[0].int()
    return pts, rois, pb, rb
