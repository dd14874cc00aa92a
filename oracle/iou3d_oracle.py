"""CPU restatement of the rotated BEV overlap / IoU / NMS of mmdet3d/ops/iou3d (iou3d_utils.py, src/iou3d.cpp, src/iou3d_kernel.cu) and of
box3d_multiclass_nms (core/post_processing/box3d_nms.py:10-143), in float64.

Boxes are [x1, y1, x2, y2, r].  Corners (x1,y1), (x2,y1), (x2,y2), (x1,y2) are turned about the box centre by
(dx cos r + dy sin r, -dx sin r + dy cos r) (iou3d_kernel.cu:111-119,158-174).  The overlap is the area of b's rectangle clipped by the
four side half-planes of a's rectangle (Sutherland-Hodgman, vectorised over box pairs), iou = overlap / max(sa + sb - overlap, 1e-8)
with s = (x2 - x1)(y2 - y1) (:244-251); the axis-aligned IoU of nms_normal ignores r (:335-343).  The greedy scan is iou3d.cpp:130-143
over the IoU matrix: in score order, a box is kept unless an earlier kept box has IoU > thresh with it.  Pairs whose circumscribed circles
are apart are 0 without clipping (the reference returns exactly 0 there too)."""
import math

import numpy as np
import torch

CHUNK = 100_000


def corners(boxes):
    """float64 [N, 4, 2] world corners, counter-clockwise for x2 > x1, y2 > y1"""
    b = np.asarray(boxes, dtype=np.float64).reshape(-1, 5)
    x1, y1, x2, y2, r = b.T
    cx, cy = (x1 + x2) / 2, (y1 + y2) / 2
    c, s = np.cos(r), np.sin(r)
    lx = np.stack([x1, x2, x2, x1], 1) - cx[:, None]
    ly = np.stack([y1, y1, y2, y2], 1) - cy[:, None]
    return np.stack([lx * c[:, None] + ly * s[:, None] + cx[:, None], -lx * s[:, None] + ly * c[:, None] + cy[:, None]], 2)


def _clip(X, Y, n, px, py, qx, qy, sign):
    """clip polygons (X, Y [P, K], n valid vertices) by the half-plane left of p->q (times sign) -> (X, Y, n) with K = 8 slots"""
    P, K = X.shape
    k = np.arange(K)[None, :]
    valid = k < n[:, None]
    nxt = np.where(k + 1 < n[:, None], k + 1, 0)
    Xn, Yn = np.take_along_axis(X, nxt, 1), np.take_along_axis(Y, nxt, 1)
    ex, ey = (qx - px)[:, None], (qy - py)[:, None]
    d0 = sign[:, None] * (ex * (Y - py[:, None]) - ey * (X - px[:, None]))     # >= 0 inside
    d1 = sign[:, None] * (ex * (Yn - py[:, None]) - ey * (Xn - px[:, None]))
    in0, in1 = d0 >= 0, d1 >= 0
    t = np.divide(d0, d0 - d1, out=np.zeros_like(d0), where=(in0 != in1))
    ix, iy = X + t * (Xn - X), Y + t * (Yn - Y)
    # every vertex emits itself (if inside) then the crossing of its outgoing edge (if the edge crosses)
    OX = np.stack([X, ix], 2).reshape(P, 2 * K)
    OY = np.stack([Y, iy], 2).reshape(P, 2 * K)
    ok = np.stack([valid & in0, valid & (in0 != in1)], 2).reshape(P, 2 * K)
    order = np.argsort(~ok, axis=1, kind="stable")
    OX, OY = np.take_along_axis(OX, order, 1)[:, :8], np.take_along_axis(OY, order, 1)[:, :8]
    return OX, OY, np.minimum(ok.sum(1), 8)


def _area(X, Y, n):
    K = X.shape[1]
    k = np.arange(K)[None, :]
    nxt = np.where(k + 1 < n[:, None], k + 1, 0)
    Xn, Yn = np.take_along_axis(X, nxt, 1), np.take_along_axis(Y, nxt, 1)
    return np.abs(np.where(k < n[:, None], X * Yn - Xn * Y, 0.0).sum(1)) / 2


def overlap_pairs(a, b):
    """float64 overlap area of box a[i] with box b[i] (both [P, 5])"""
    a, b = np.asarray(a, np.float64).reshape(-1, 5), np.asarray(b, np.float64).reshape(-1, 5)
    out = np.zeros(a.shape[0])
    for s in range(0, a.shape[0], CHUNK):
        ca, cb = corners(a[s:s + CHUNK]), corners(b[s:s + CHUNK])
        P = ca.shape[0]
        sa = (a[s:s + CHUNK, 2] - a[s:s + CHUNK, 0]) * (a[s:s + CHUNK, 3] - a[s:s + CHUNK, 1])
        sign = np.where(sa >= 0, 1.0, -1.0)                 # a flipped box (x2 < x1 xor y2 < y1) runs clockwise
        X = np.zeros((P, 8))
        Y = np.zeros((P, 8))
        X[:, :4], Y[:, :4] = cb[:, :, 0], cb[:, :, 1]
        n = np.full(P, 4)
        for e in range(4):
            p, q = ca[:, e], ca[:, (e + 1) % 4]
            X, Y, n = _clip(X, Y, n, p[:, 0], p[:, 1], q[:, 0], q[:, 1], sign)
        area = _area(X, Y, n)
        sb = (b[s:s + CHUNK, 2] - b[s:s + CHUNK, 0]) * (b[s:s + CHUNK, 3] - b[s:s + CHUNK, 1])
        out[s:s + CHUNK] = np.where((sa != 0) & (sb != 0), area, 0.0)     # a zero-area box has no inside
    return out


def _areas(b):
    return (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])


def candidate_pairs(a, b, upper=False):
    """(i, j) whose circumscribed circles meet (every pair with a non-zero overlap is among them); upper: j > i only"""
    a, b = np.asarray(a, np.float64).reshape(-1, 5), np.asarray(b, np.float64).reshape(-1, 5)
    ca, cb = (a[:, :2] + a[:, 2:4]) / 2, (b[:, :2] + b[:, 2:4]) / 2
    ra, rb = np.hypot(a[:, 2] - a[:, 0], a[:, 3] - a[:, 1]) / 2, np.hypot(b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]) / 2
    I, J = [], []
    rows = max(1, 4_000_000 // max(b.shape[0], 1))
    for s in range(0, a.shape[0], rows):
        d2 = ((ca[s:s + rows, None, :] - cb[None, :, :]) ** 2).sum(-1)
        hit = d2 <= (ra[s:s + rows, None] + rb[None, :]) ** 2 * (1 + 1e-9) + 1e-12
        if upper:
            hit &= np.arange(s, s + hit.shape[0])[:, None] < np.arange(b.shape[0])[None, :]
        i, j = np.nonzero(hit)
        I.append(i + s)
        J.append(j)
    if not I:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(I).astype(np.int64), np.concatenate(J).astype(np.int64)


def iou_from_overlap(a, b, ov):
    return ov / np.maximum(_areas(a) + _areas(b) - ov, 1e-8)


def normal_iou_pairs(a, b):
    left, right = np.maximum(a[:, 0], b[:, 0]), np.minimum(a[:, 2], b[:, 2])
    top, bottom = np.maximum(a[:, 1], b[:, 1]), np.minimum(a[:, 3], b[:, 3])
    inter = np.maximum(right - left, 0) * np.maximum(bottom - top, 0)
    return inter / np.maximum(_areas(a) + _areas(b) - inter, 1e-8)


def pair_values(boxes_a, boxes_b, what="iou", upper=False):
    """(i, j, value) over the candidate pairs; every other pair is exactly 0 (what: 'iou', 'overlap' or 'normal')"""
    a = np.asarray(torch.as_tensor(boxes_a).double().numpy()).reshape(-1, 5)
    b = np.asarray(torch.as_tensor(boxes_b).double().numpy()).reshape(-1, 5)
    i, j = candidate_pairs(a, b, upper)      # the circumscribed circle also holds the axis-aligned rectangle
    if what == "normal":
        return i, j, normal_iou_pairs(a[i], b[j])
    ov = overlap_pairs(a[i], b[j])
    return i, j, (ov if what == "overlap" else iou_from_overlap(a[i], b[j], ov))


def _matrix(boxes_a, boxes_b, what):
    M, N = len(boxes_a), len(boxes_b)
    out = np.zeros((M, N))
    if M and N:
        i, j, v = pair_values(boxes_a, boxes_b, what)
        out[i, j] = v
    return torch.from_numpy(out)


def boxes_overlap_bev(boxes_a, boxes_b):
    """float64 [M, N] overlap areas"""
    return _matrix(boxes_a, boxes_b, "overlap")


def boxes_iou_bev(boxes_a, boxes_b):
    """float64 [M, N] rotated IoU (iou3d_utils.py:12-28)"""
    return _matrix(boxes_a, boxes_b, "iou")


def nms_sorted(boxes, thresh, rotated=True):
    """the greedy scan of iou3d.cpp:130-143 over boxes already in score order -> kept positions (int64)"""
    n = len(boxes)
    if n == 0:
        return torch.zeros(0, dtype=torch.long)
    return greedy_scan(n, *pair_values(boxes, boxes, "iou" if rotated else "normal", upper=True), thresh)


def greedy_scan(n, i, j, v, thresh):
    """the scan over upper-triangle pair values (i < j, value v; absent pairs are 0) of n boxes in score order"""
    if n == 0:
        return torch.zeros(0, dtype=torch.long)
    sup = v > thresh
    i, j = i[sup], j[sup]
    order = np.argsort(i, kind="stable")
    i, j = i[order], j[order]
    start = np.searchsorted(i, np.arange(n + 1))
    removed = np.zeros(n, bool)
    keep = []
    for r in range(n):
        if not removed[r]:
            keep.append(r)
            removed[j[start[r]:start[r + 1]]] = True
    return torch.tensor(keep, dtype=torch.long)


def nms_gpu(boxes, scores, thresh, pre_maxsize=None, post_max_size=None):
    """iou3d_utils.py:31-56 on the CPU"""
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    keep = order[nms_sorted(boxes[order], thresh, True)].contiguous()
    if post_max_size is not None:
        keep = keep[:post_max_size]
    return keep


def nms_normal_gpu(boxes, scores, thresh):
    """iou3d_utils.py:106-124 on the CPU"""
    order = scores.sort(0, descending=True)[1]
    return order[nms_sorted(boxes[order], thresh, False)].contiguous()


def box3d_multiclass_nms(mlvl_bboxes, mlvl_bboxes_for_nms, mlvl_scores, score_thr, max_num, cfg, mlvl_dir_scores=None,
                         mlvl_attr_scores=None, mlvl_bboxes2d=None, nms_gpu=nms_gpu, nms_normal_gpu=nms_normal_gpu):
    """box3d_nms.py:10-143 restated (per-class loop, class-ordered concatenation, max_num cut by scores.sort(descending=True), the
    empty-result shapes); nms_gpu / nms_normal_gpu may be swapped for another implementation of the same functions"""
    num_classes = mlvl_scores.shape[1] - 1
    bboxes, scores, labels, dir_scores, attr_scores, bboxes2d = [], [], [], [], [], []
    for i in range(num_classes):
        cls_score_thr = score_thr[i] if isinstance(score_thr, (list, tuple)) else score_thr
        nms_thr = cfg.nms_thr
        if isinstance(nms_thr, (list, tuple)):
            nms_thr = nms_thr[i]
        cls_inds = mlvl_scores[:, i] > cls_score_thr
        if not cls_inds.any():
            continue
        _scores = mlvl_scores[cls_inds, i]
        _bboxes_for_nms = mlvl_bboxes_for_nms[cls_inds, :]
        nms_func = nms_gpu if cfg.use_rotate_nms else nms_normal_gpu
        if nms_thr is None:
            selected = torch.arange(len(_scores), dtype=torch.long, device=_scores.device)
        else:
            selected = nms_func(_bboxes_for_nms, _scores, nms_thr)
        bboxes.append(mlvl_bboxes[cls_inds, :][selected])
        scores.append(_scores[selected])
        labels.append(mlvl_bboxes.new_full((len(selected),), i, dtype=torch.long))
        if mlvl_dir_scores is not None:
            dir_scores.append(mlvl_dir_scores[cls_inds][selected])
        if mlvl_attr_scores is not None:
            attr_scores.append(mlvl_attr_scores[cls_inds][selected])
        if mlvl_bboxes2d is not None:
            bboxes2d.append(mlvl_bboxes2d[cls_inds][selected])
    if bboxes:
        bboxes, scores, labels = torch.cat(bboxes), torch.cat(scores), torch.cat(labels)
        dir_scores = torch.cat(dir_scores) if mlvl_dir_scores is not None else None
        attr_scores = torch.cat(attr_scores) if mlvl_attr_scores is not None else None
        bboxes2d = torch.cat(bboxes2d) if mlvl_bboxes2d is not None else None
        if bboxes.shape[0] > max_num:
            inds = scores.sort(descending=True)[1][:max_num]
            bboxes, labels, scores = bboxes[inds, :], labels[inds], scores[inds]
            dir_scores = dir_scores[inds] if dir_scores is not None else None
            attr_scores = attr_scores[inds] if attr_scores is not None else None
            bboxes2d = bboxes2d[inds] if bboxes2d is not None else None
    else:
        bboxes = mlvl_scores.new_zeros((0, mlvl_bboxes.size(-1)))
        scores = mlvl_scores.new_zeros((0,))
        labels = mlvl_scores.new_zeros((0,), dtype=torch.long)
        dir_scores = mlvl_scores.new_zeros((0,)) if mlvl_dir_scores is not None else None
        attr_scores = mlvl_scores.new_zeros((0,)) if mlvl_attr_scores is not None else None
        bboxes2d = mlvl_scores.new_zeros((0, 4)) if mlvl_bboxes2d is not None else None
    results = (bboxes, scores, labels)
    for extra, given in ((dir_scores, mlvl_dir_scores), (attr_scores, mlvl_attr_scores), (bboxes2d, mlvl_bboxes2d)):
        if given is not None:
            results = results + (extra,)
    return results


# ---- synthetic inputs -------------------------------------------------------------------------------------------------------------
def synth_boxes(seed, n, spread=75.0, objects=None, jitter=0.3):
    """fp32 [n, 5] xyxyr boxes: centres in +-spread m, sizes 0.2-12 m, yaw in [-pi, pi].  objects=K: an FSD-like dense case, n proposals
    around K objects (centre jitter `jitter` m, size jitter 10 %, yaw jitter 0.2 rad)."""
    g = torch.Generator().manual_seed(seed)
    if objects is None:
        c = (torch.rand(n, 2, generator=g) * 2 - 1) * spread
        wl = 0.2 + torch.rand(n, 2, generator=g) * 11.8
        r = (torch.rand(n, generator=g) * 2 - 1) * math.pi
    else:
        oc = (torch.rand(objects, 2, generator=g) * 2 - 1) * spread
        owl = 0.5 + torch.rand(objects, 2, generator=g) * 5.5
        orr = (torch.rand(objects, generator=g) * 2 - 1) * math.pi
        k = torch.randint(0, objects, (n,), generator=g)
        c = oc[k] + torch.randn(n, 2, generator=g) * jitter
        wl = owl[k] * (1 + 0.1 * torch.randn(n, 2, generator=g)).clamp(min=0.3)
        r = orr[k] + 0.2 * torch.randn(n, generator=g)
    return torch.cat([c - wl / 2, c + wl / 2, r[:, None]], 1).float()


def distinct_scores(seed, n):
    """n distinct fp32 scores in (0, 1), randomly ordered"""
    g = torch.Generator().manual_seed(seed)
    return ((torch.randperm(n, generator=g).double() + 0.5) / max(n, 1)).float()


def drop_near_threshold(boxes, threshs, margin=1e-4, rotated=True):
    """boxes minus every box that has a pair with an IoU within `margin` of one of `threshs` (removing boxes changes no other
    pair's IoU, so the rest compares well-defined at those thresholds) -> kept row indices"""
    i, j, v = pair_values(boxes, boxes, "iou" if rotated else "normal", upper=True)
    bad = np.zeros(len(boxes), bool)
    for t in threshs:
        bad[j[np.abs(v - t) < margin]] = True   # the later box of every near pair
    return torch.from_numpy(np.nonzero(~bad)[0])


def special_boxes():
    """fp32 [K, 5] boxes whose pairs hit the geometry's edge cases: identical and nested boxes, shared and collinear edges, corners
    exactly on edges, r in {0, +-pi/2, pi}, near-parallel edges (the reference's |s5 - s1| <= EPS branch), zero-area boxes, and a far
    copy 70 m from the origin"""
    h = math.pi / 2
    rows = [
        [0, 0, 4, 2, 0.3], [0, 0, 4, 2, 0.3],                  # identical
        [1, 0.5, 3, 1.5, 0.3],                                 # nested in the two above
        [4, 0, 8, 2, 0.0], [0, 0, 4, 2, 0.0],                  # shared edge x = 4 (touching)
        [2, 0, 6, 2, 0.0], [2, 1, 6, 3, 0.0],                  # collinear edges, half overlaps
        [1, -1, 3, 1, math.pi / 2],                            # turned square: corners on the others' edges
        [3, 1, 5, 3, 0.0], [-2, -1, 2, 1, h], [-2, -1, 2, 1, -h], [-2, -1, 2, 1, math.pi],
        [0, 0, 4, 2, 0.3 + 1e-7], [0.001, 0, 4.001, 2, 0.3 - 2e-7],   # near-parallel edges
        [0, 0, 4, 2, 1e-6], [0, 1e-5, 4, 2 + 1e-5, 0.0],
        [2, 1, 2, 1, 0.0], [1, 0, 3, 0, 0.2], [0, 0, 0, 5, 0.7],      # zero area: a point and two segments
        [70.0, 70.0, 74.0, 72.0, 0.3], [70.0, 70.0, 74.0, 72.0, 0.3], [71.0, 70.5, 73.0, 71.5, 1.2],
        [-75.0, 30.0, -63.0, 42.0, -2.9], [-74.9, 30.1, -62.9, 42.1, -2.9 + 1e-7],
    ]
    return torch.tensor(rows, dtype=torch.float32)
