"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

CPU restatement of mmdet3d/ops/roiaware_pool3d: points_in_boxes_gpu / points_in_boxes_batch (src/points_in_boxes_cuda.cu) and
RoIAwarePool3d forward / backward (src/roiaware_pool3d_kernel.cu), plus Single3DRoIAwareExtractor's per-sample loop
(models/roi_heads/roi_extractors/single_roiaware_extractor.py:31-53).  The box test is roi_pool_oracle.box_test (pinned to the
reference's points_in_boxes_cpu by tests/test_oracle_roi_pool_vs_reference.py); results are laid out as the reference lays them out:
pts_idx_of_voxels [R, ox, oy, oz, m] (slot 0 = count), argmax [R, ox, oy, oz, C], pooled [R, ox, oy, oz, C]."""
import torch

from oracle.roi_pool_oracle import box_test


def membership(pts, boxes, chunk=32):
    """inside [T, M] bool, plus local x / y [T, M] fp32, for pts [M, 3] and boxes [T, 7]"""
    pts, boxes = pts.float(), boxes.float()
    ins, lxs, lys = [], [], []
    for k0 in range(0, boxes.shape[0], chunk):
        inside, lx, ly, _ = box_test(pts, boxes[k0:k0 + chunk])
        ins.append(inside), lxs.append(lx), lys.append(ly)
    if not ins:
        z = torch.zeros((0, pts.shape[0]))
        return z.bool(), z, z
    return torch.cat(ins), torch.cat(lxs), torch.cat(lys)


def points_in_boxes_gpu(points, boxes):
    """[B, M, 3], [B, T, 7] -> int32 [B, M]: the lowest box index holding the point, else -1"""
    B, M, _ = points.shape
    out = torch.full((B, M), -1, dtype=torch.int32)
    for b in range(B):
        inside = membership(points[b], boxes[b])[0]
        if inside.shape[0] and M:
            out[b] = torch.where(inside.any(0), inside.int().argmax(0), -1).int()   # argmax: the first maximal index
    return out


def points_in_boxes_batch(points, boxes):
    """[B, M, 3], [B, T, 7] -> int32 [B, M, T] of 1 / 0"""
    B, M, _ = points.shape
    out = torch.zeros((B, M, boxes.shape[1]), dtype=torch.int32)
    for b in range(B):
        out[b] = membership(points[b], boxes[b])[0].t().int()
    return out


def _cvt_index(v, o):
    """roiaware_pool3d_kernel.cu:83-89: unsigned idx = int(v) (CUDA's cvt.rzi: truncation, NaN -> 0, saturating), min(max(idx, 0),
    o - 1) on the unsigned value, so a negative index lands in cell o - 1"""
    t = torch.nan_to_num(torch.trunc(v.double()), nan=0.0).clamp(-2.0 ** 31, 2.0 ** 31 - 1).long()
    return torch.where(t < 0, torch.full_like(t, o - 1), t.clamp(max=o - 1))


def voxel_index(rois, lx, ly, z, out_size):
    """flat voxel (x * oy + y) * oz + z of every (RoI, point): lx / ly [R, N] fp32 local coordinates, z [N]; the fp32 steps
    x_res = l / ox, idx = int((lx + l / 2) / x_res), z from the bottom"""
    ox, oy, oz = out_size
    w, l, h = rois[:, 3:4], rois[:, 4:5], rois[:, 5:6]
    xi = _cvt_index((lx + l / 2) / (l / ox), ox)
    yi = _cvt_index((ly + w / 2) / (w / oy), oy)
    zi = _cvt_index((z[None] - rois[:, 2:3]) / (h / oz), oz)
    return (xi * oy + yi) * oz + zi


def out_size3(out_size):
    return (out_size,) * 3 if isinstance(out_size, int) else tuple(out_size)


def roiaware_pool3d(rois, pts, pts_feature, out_size, max_pts_per_voxel, mode, rois_batch=None, pts_batch=None):
    """forward: returns pooled, argmax (-1 where nothing was selected; zeros in avg mode, as the reference leaves its buffer),
    pts_idx_of_voxels.  mode 0 = max, 1 = avg.  With batch ids a point pairs only with RoIs of its own sample."""
    ox, oy, oz = out_size3(out_size)
    nvox = ox * oy * oz
    rois, pts, feats = rois.float(), pts.float(), pts_feature.float()
    R, N, C = rois.shape[0], pts.shape[0], feats.shape[1]
    m = max_pts_per_voxel
    inside, lx, ly = membership(pts, rois)
    if rois_batch is not None:
        inside &= rois_batch.long()[:, None] == pts_batch.long()[None]
    r_idx, p_idx = inside.nonzero(as_tuple=True)                          # RoI-major, points ascending
    vox = voxel_index(rois, lx, ly, pts[:, 2], (ox, oy, oz))[r_idx, p_idx] if r_idx.numel() else r_idx
    key = r_idx * nvox + vox
    order = torch.sort(key, stable=True).indices
    key, pnt = key[order], p_idx[order]
    uniq, counts = torch.unique_consecutive(key, return_counts=True)
    start = torch.repeat_interleave(torch.cumsum(counts, 0) - counts, counts)
    rank = torch.arange(key.numel()) - start
    keep = rank < m - 1
    key, pnt, rank = key[keep], pnt[keep], rank[keep]
    pidx = torch.zeros((R * nvox, m), dtype=torch.int32)
    kept_cnt = torch.clamp(counts, max=m - 1)
    pidx[uniq, 0] = kept_cnt.int()
    pidx[key, rank + 1] = pnt.int()
    pooled = torch.zeros((R * nvox, C))
    argmax = torch.full((R * nvox, C), -1 if mode == 0 else 0, dtype=torch.int32)
    best = torch.full((R * nvox, C), -float("inf"))
    arg = torch.full((R * nvox, C), -1, dtype=torch.long)
    acc = torch.zeros((R * nvox, C))
    for j in range(int(rank.max()) + 1 if rank.numel() else 0):          # ascending point order inside every voxel
        sel = rank == j
        g, x = key[sel], feats[pnt[sel]]
        if mode == 0:
            upd = x > best[g]
            best[g] = torch.where(upd, x, best[g])
            arg[g] = torch.where(upd, pnt[sel][:, None].expand_as(x), arg[g])
        else:
            acc[g] = acc[g] + x
    if mode == 0:
        hit = arg >= 0
        pooled[hit] = best[hit]
        argmax = arg.int()
    else:
        cnt = pidx[:, 0].float()[:, None]
        nz = (cnt > 0).expand_as(acc)
        pooled[nz] = (acc / cnt.clamp(min=1))[nz]
    shp = (R, ox, oy, oz)
    return pooled.view(*shp, C), argmax.view(*shp, C), pidx.view(*shp, m)


def roiaware_pool3d_backward(pts_idx_of_voxels, argmax, grad_out, num_pts, mode):
    """roiaware_pool3d_kernel.cu:288-352 with the contributions to a point added in (RoI, voxel) order: grad_in [num_pts, C] fp32"""
    R = grad_out.shape[0]
    C = grad_out.shape[-1]
    go = grad_out.float().reshape(R, -1, C)
    grad_in = torch.zeros((num_pts, C))
    m = pts_idx_of_voxels.shape[-1]
    for r in range(R):                                                   # inside one RoI a point sits in one voxel
        if mode == 0:
            a = argmax[r].reshape(-1, C).long()
            v, c = (a >= 0).nonzero(as_tuple=True)
            grad_in.index_put_((a[v, c], c), go[r, v, c] * 1, accumulate=True)
        else:
            pi = pts_idx_of_voxels[r].reshape(-1, m).long()
            cnt = pi[:, 0]
            v, s = (torch.arange(m - 1)[None] < cnt[:, None]).nonzero(as_tuple=True)
            cur = 1.0 / torch.clamp(cnt.float(), min=1.0)
            grad_in.index_put_((pi[v, s + 1],), go[r, v] * cur[v][:, None], accumulate=True)
    return grad_in


def expand_state(slot, voff, pidx, argmax, counts, R, out_size, m, C):
    """this library's compact RoIAwarePool3d state (voxel slots, kept-point CSR, [occupied, C] argmax) in the reference's dense layout:
    pts_idx_of_voxels [R, ox, oy, oz, m] and argmax [R, ox, oy, oz, C] (-1 where nothing was selected)"""
    ox, oy, oz = out_size3(out_size)
    V, K = int(counts[0]), int(counts[1])
    slot, voff, pidx = slot[:V].long(), voff[:V + 1].long(), pidx[:K].long()
    dense = torch.zeros((R * ox * oy * oz, m), dtype=torch.int32)
    cnt = voff[1:] - voff[:-1]
    dense[slot, 0] = cnt.int()
    g = torch.repeat_interleave(torch.arange(V), cnt)
    rank = torch.arange(K) - voff[:-1][g]
    dense[slot[g], rank + 1] = pidx.int()
    am = torch.full((R * ox * oy * oz, C), -1, dtype=torch.int32)
    if argmax is not None:
        am[slot] = argmax[:V].int()
    return dense.view(R, ox, oy, oz, m), am.view(R, ox, oy, oz, C)


def single_roiaware_extractor(feats, coordinate, batch_inds, rois, out_size, max_pts_per_voxel, mode):
    """single_roiaware_extractor.py:31-53: pooled features of every sample's RoIs, sample after sample"""
    out = []
    for b in range(int(batch_inds.max()) + 1):
        ri, ci = rois[..., 0].int() == b, batch_inds.int() == b
        out.append(roiaware_pool3d(rois[..., 1:][ri], coordinate[ci], feats[ci], out_size, max_pts_per_voxel, mode)[0])
    return torch.cat(out, 0)


def golden_inputs():
    """the inputs of tests/golden/roiaware_pool3d.npz (oracle/make_golden_roiaware.py): 6 overlapping RoIs, points on their faces, a
    crowded voxel, out_size (6, 4, 3), m = 8, C = 5 features with ties and NaN / -inf entries; and a 2-sample points_in_boxes batch"""
    g = torch.Generator().manual_seed(2024)
    rois = torch.tensor([[0.0, 0.0, -1.0, 2.0, 4.0, 1.5, 0.0],
                         [0.5, 0.3, -1.2, 2.2, 4.4, 1.8, 0.3],       # overlaps RoI 0
                         [6.0, -2.0, -0.5, 1.0, 1.0, 2.0, -1.5707964],
                         [6.2, -2.1, -0.6, 1.2, 1.4, 2.1, 1.2],      # overlaps RoI 2
                         [-5.0, 4.0, 0.0, 3.0, 3.0, 3.0, 2.5],
                         [20.0, 20.0, 0.0, 1.0, 1.0, 1.0, 0.0]])     # empty
    pts = [rois[r, :3] + (torch.rand((60, 3), generator=g) - 0.5) * torch.stack([rois[r, 4], rois[r, 3], rois[r, 5]]) * 1.2
           + torch.tensor([0.0, 0.0, 1.0]) * rois[r, 5] / 2 for r in range(5)]
    # faces: the exact +-l/2, +-w/2 and bottom / top values of axis-aligned RoI 2 (yaw -pi/2: local axes = world axes up to rounding)
    cx, cy, zb, w, l, h = rois[2, :6].tolist()
    face = torch.tensor([[cx + l / 2, cy, zb + h / 2], [cx - l / 2, cy, zb + h / 2], [cx, cy + w / 2, zb + h / 2], [cx, cy - w / 2, zb + h / 2],
                         [cx, cy, zb], [cx, cy, zb + h], [cx + 0.1, cy + 0.1, zb], [cx - 0.2, cy, zb + h]])
    crowd = torch.tensor([0.1, 0.1, -0.5]) + torch.rand((20, 3), generator=g) * 0.05   # > m - 1 points in one voxel of RoIs 0 and 1
    pts = torch.cat(pts + [face, crowd]).float()
    feats = torch.randn((pts.shape[0], 5), generator=g)
    feats[::7, 1] = feats[3, 1]                                          # ties
    feats[::11, 2] = float("nan")
    feats[::13, 3] = -float("inf")
    grad = torch.randn((rois.shape[0], 6, 4, 3, 5), generator=g)
    pib_boxes = torch.stack([rois, torch.cat([rois[:4], torch.zeros((2, 7))])])   # sample 1: two zero-size padding boxes
    pib_pts = torch.stack([pts[:200], pts[-200:]])
    return dict(rois=rois, pts=pts, feats=feats, grad=grad, pib_boxes=pib_boxes.contiguous(), pib_pts=pib_pts.contiguous(),
                out_size=(6, 4, 3), m=8)
