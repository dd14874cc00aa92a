"""Python face of the op surface the reference exports from `mmdet3d.ops`
(mmdet3d/ops/__init__.py:23-30), backed by libsstb200 (CUDA, sm_90a).  Same names, argument meaning
and error behaviour; no CPU path - CPU tensors raise.

    Voxelization / voxelization       ops/voxel/voxelize.py:11-130          (dynamic branch only, V1)
    DynamicScatter / dynamic_scatter  ops/voxel/scatter_points.py:9-110      (V2, V3)
    scatter_v2                        ops/sst/sst_ops.py:151-182             (V5)
    get_inner_win_inds                ops/sst/sst_ops.py:244-264             (B2)
    get_window_coors, make_continuous_inds, get_flat2win_inds(_v2), flat2window(_v2), window2flat(_v2)
                                      ops/sst/sst_ops.py:27-149,266-331      (B1, B4, B6)
    build_mlp, get_activation(_layer) ops/sst/sst_ops.py:334-392             (S3)
    dynamic_point_pool(_mixed)        ops/dynamic_point_pool_op.py:9-113     (FSD RoI point pooling)
    boxes_iou_bev, boxes_overlap_bev, nms_gpu, nms_normal_gpu
                                      ops/iou3d/iou3d_utils.py               (rotated BEV IoU / NMS)
    box3d_multiclass_nms              core/post_processing/box3d_nms.py:10-143
    points_in_boxes_gpu, points_in_boxes_batch, RoIAwarePool3d
                                      ops/roiaware_pool3d                    (box membership, RoI-aware pooling)
    deform_conv2d, DeformConv2dFunction
                                      mmcv.ops.deform_conv (1.3.8-1.4.0)    (CenterHead's DCN)
    anchor3d_targets, anchor_focal_loss, anchor_reg_dir_loss
                                      models/dense_heads/anchor3d_head.py, train_mixins.py (Anchor3DHead training)
    voteseg_targets, voteseg_loss     models/decode_heads/segmentation_head.py:107-283 (VoteSegHead training)
    cluster_head_targets, cluster_head_loss, multiclass_nms_groups
                                      models/dense_heads/sparse_cluster_head_v2.py (SparseClusterHeadV2 training and proposals)
"""
import ctypes as C
import math

import numpy as np
import torch
import torch.nn as nn
from torch.autograd import Function

from . import _lib as L

_REDUCE = {"sum": 0, "mean": 1, "max": 2}


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.SSTB200Error("sst_b200 ops need CUDA tensors (H100); there is no CPU implementation")


# ----------------------------------------------------------------------------------------------
# V1 voxelization
# ----------------------------------------------------------------------------------------------
def dynamic_voxelize(points, coors, voxel_size, coors_range, NDim=3):
    """voxel_layer.dynamic_voxelize (ops/voxel/src/voxelization.h:72-88): fills caller-allocated `coors`."""
    assert NDim == 3
    _need_cuda(points, coors)
    assert points.dtype == torch.float32 and coors.dtype == torch.int32
    assert points.is_contiguous() and coors.is_contiguous(), "points/coors must be contiguous"
    c = L.ctx(points.device)
    L.check(c, L.lib().sstb200_dynamic_voxelize(
        c, points.data_ptr(), points.shape[0], points.shape[1], L.arr(C.c_float, [float(v) for v in voxel_size]),
        L.arr(C.c_float, [float(v) for v in coors_range]), coors.data_ptr()))


def hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size, coors_range, max_points, max_voxels, NDim=3):
    """voxel_layer.hard_voxelize (ops/voxel/src/voxelization.h:51-70): fills the caller's zero-initialised buffers, returns the
    number of voxels (int, one stream sync like the reference)."""
    assert NDim == 3
    _need_cuda(points, voxels, coors, num_points_per_voxel)
    assert points.dtype == torch.float32 and voxels.dtype == torch.float32
    assert coors.dtype == torch.int32 and num_points_per_voxel.dtype == torch.int32
    for t in (points, voxels, coors, num_points_per_voxel):
        assert t.is_contiguous()
    assert voxels.shape == (max_voxels, max_points, points.shape[1]) and coors.shape == (max_voxels, 3)
    num_dev = torch.empty((1,), dtype=torch.int32, device=points.device)
    num = C.c_int32(0)
    c = L.ctx(points.device)
    L.check(c, L.lib().sstb200_hard_voxelize(
        c, points.data_ptr(), points.shape[0], points.shape[1], L.arr(C.c_float, [float(v) for v in voxel_size]),
        L.arr(C.c_float, [float(v) for v in coors_range]), int(max_points), int(max_voxels), voxels.data_ptr(), coors.data_ptr(),
        num_points_per_voxel.data_ptr(), num_dev.data_ptr(), C.byref(num)))
    return num.value


class _Voxelization(Function):
    """ops/voxel/voxelize.py:11-72."""

    @staticmethod
    def forward(ctx, points, voxel_size, coors_range, max_points=35, max_voxels=20000):
        if max_points == -1 or max_voxels == -1:
            coors = points.new_zeros(size=(points.size(0), 3), dtype=torch.int)
            dynamic_voxelize(points.contiguous(), coors, voxel_size, coors_range, 3)
            return coors
        points = points.contiguous()
        voxels = points.new_zeros(size=(max_voxels, max_points, points.size(1)))
        coors = points.new_zeros(size=(max_voxels, 3), dtype=torch.int)
        num_points_per_voxel = points.new_zeros(size=(max_voxels,), dtype=torch.int)
        voxel_num = hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size, coors_range, max_points, max_voxels, 3)
        return voxels[:voxel_num], coors[:voxel_num], num_points_per_voxel[:voxel_num]


voxelization = _Voxelization.apply


class Voxelization(nn.Module):
    """ops/voxel/voxelize.py:77-130."""

    def __init__(self, voxel_size, point_cloud_range, max_num_points, max_voxels=20000):
        super().__init__()
        self.voxel_size = voxel_size
        self.point_cloud_range = point_cloud_range
        self.max_num_points = max_num_points
        self.max_voxels = max_voxels if isinstance(max_voxels, tuple) else (max_voxels, max_voxels)
        pcr = torch.tensor(point_cloud_range, dtype=torch.float32)
        grid = torch.round((pcr[3:] - pcr[:3]) / torch.tensor(voxel_size, dtype=torch.float32)).long()
        self.grid_size = grid
        self.pcd_shape = [*grid[:2], 1][::-1]

    def forward(self, input):
        mv = self.max_voxels[0] if self.training else self.max_voxels[1]
        return voxelization(input, self.voxel_size, self.point_cloud_range, self.max_num_points, mv)

    def __repr__(self):
        return (f"{self.__class__.__name__}(voxel_size={self.voxel_size}, point_cloud_range="
                f"{self.point_cloud_range}, max_num_points={self.max_num_points}, max_voxels={self.max_voxels})")


# ----------------------------------------------------------------------------------------------
# V2/V3 DynamicScatter
# ----------------------------------------------------------------------------------------------
def dynamic_point_to_voxel_forward(feats, coors, reduce_type, coor_bounds=None):
    """voxel_layer.dynamic_point_to_voxel_forward -> [reduced_feats, out_coors, coors_map, reduce_count].
    `coor_bounds` = (lo[3], hi[3]) of the valid coordinates if the caller knows the grid (saves one reduction
    + sync); otherwise they are measured from `coors`."""
    _need_cuda(feats, coors)
    assert feats.dtype == torch.float32, "fp32 feats only"
    assert coors.dtype == torch.int32 and coors.dim() == 2 and coors.shape[1] == 3
    assert feats.is_contiguous() and coors.is_contiguous(), "feats/coors must be contiguous"
    P, Cc = feats.shape
    dev = feats.device
    if P == 0:
        return [feats.clone().detach(), coors.clone().detach(), coors.new_empty((0,), dtype=torch.int32),
                coors.new_empty((0,), dtype=torch.int32)]
    if coor_bounds is None:
        hi = coors.amax(0).clamp(min=0).tolist()
        lo = [0, 0, 0]
    else:
        lo, hi = coor_bounds
    reduced = torch.empty((P, Cc), dtype=torch.float32, device=dev)
    out_coors = torch.empty((P, 3), dtype=torch.int32, device=dev)
    cmap = torch.empty((P,), dtype=torch.int32, device=dev)
    count = torch.empty((P,), dtype=torch.int32, device=dev)
    num_dev = torch.empty((1,), dtype=torch.int32, device=dev)
    num_host = C.c_int32(0)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_dynamic_point_to_voxel_forward(
        c, feats.data_ptr(), coors.data_ptr(), P, Cc, _REDUCE[reduce_type], L.arr(C.c_int32, [int(v) for v in lo]),
        L.arr(C.c_int32, [int(v) for v in hi]), reduced.data_ptr(), out_coors.data_ptr(), cmap.data_ptr(),
        count.data_ptr(), num_dev.data_ptr(), C.byref(num_host)))
    M = num_host.value
    return [reduced[:M], out_coors[:M], cmap, count[:M]]


def dynamic_point_to_voxel_backward(grad_feats, grad_reduced_feats, feats, reduced_feats, coors_map, reduce_count,
                                    reduce_type):
    """voxel_layer.dynamic_point_to_voxel_backward: fills caller-allocated grad_feats."""
    _need_cuda(grad_feats, grad_reduced_feats, feats, reduced_feats, coors_map, reduce_count)
    for t in (grad_feats, grad_reduced_feats, feats, reduced_feats, coors_map, reduce_count):
        assert t.is_contiguous()
    c = L.ctx(feats.device)
    L.check(c, L.lib().sstb200_dynamic_point_to_voxel_backward(
        c, grad_feats.data_ptr(), grad_reduced_feats.data_ptr(), feats.data_ptr(), reduced_feats.data_ptr(),
        coors_map.data_ptr(), reduce_count.data_ptr(), feats.shape[0], reduced_feats.shape[0], feats.shape[1],
        _REDUCE[reduce_type]))


class _dynamic_scatter(Function):
    """ops/voxel/scatter_points.py:9-49."""

    @staticmethod
    def forward(ctx, feats, coors, reduce_type="max", coor_bounds=None):
        voxel_feats, voxel_coors, point2voxel_map, voxel_points_count = dynamic_point_to_voxel_forward(
            feats, coors, reduce_type, coor_bounds)
        ctx.reduce_type = reduce_type
        ctx.save_for_backward(feats, voxel_feats, point2voxel_map, voxel_points_count)
        ctx.mark_non_differentiable(voxel_coors)
        return voxel_feats, voxel_coors

    @staticmethod
    def backward(ctx, grad_voxel_feats, grad_voxel_coors=None):
        feats, voxel_feats, point2voxel_map, voxel_points_count = ctx.saved_tensors
        grad_feats = torch.empty_like(feats)
        dynamic_point_to_voxel_backward(grad_feats, grad_voxel_feats.contiguous(), feats, voxel_feats.contiguous(),
                                        point2voxel_map, voxel_points_count.contiguous(), ctx.reduce_type)
        return grad_feats, None, None, None


dynamic_scatter = _dynamic_scatter.apply


class DynamicScatter(nn.Module):
    """ops/voxel/scatter_points.py:52-110."""

    def __init__(self, voxel_size, point_cloud_range, average_points: bool):
        super().__init__()
        self.voxel_size = voxel_size
        self.point_cloud_range = point_cloud_range
        self.average_points = average_points
        # (z, y, x) grid of the voxelisation this layer is paired with (voxelize.py:95-100): the bitmap-rank index is
        # sized from it, so no reduction + host sync over the coordinates is needed.  Coordinates outside this grid
        # (impossible when they come from `Voxelization` with the same range) make the call fail loudly.
        self._bounds = None
        if voxel_size is not None and point_cloud_range is not None:
            r, v = point_cloud_range, voxel_size
            g = [int(math.ceil((r[3 + i] - r[i]) / v[i])) + 1 for i in range(3)]  # ceil-grid of voxelization_cpu.cpp:151-158, +1 slack
            self._bounds = ([0, 0, 0], [g[2], g[1], g[0]])

    def forward_single(self, points, coors):
        reduce = "mean" if self.average_points else "max"
        return dynamic_scatter(points.contiguous(), coors.contiguous(), reduce, self._bounds)

    def forward(self, points, coors):
        if coors.size(-1) == 3:
            return self.forward_single(points, coors)
        batch_size = int(coors[-1, 0]) + 1
        voxels, voxel_coors = [], []
        for i in range(batch_size):
            inds = torch.where(coors[:, 0] == i)
            voxel, voxel_coor = self.forward_single(points[inds], coors[inds][:, 1:])
            voxel_coors.append(nn.functional.pad(voxel_coor, (1, 0), mode="constant", value=i))
            voxels.append(voxel)
        return torch.cat(voxels, dim=0), torch.cat(voxel_coors, dim=0)

    def __repr__(self):
        return (f"{self.__class__.__name__}(voxel_size={self.voxel_size}, point_cloud_range="
                f"{self.point_cloud_range}, average_points={self.average_points})")


# ----------------------------------------------------------------------------------------------
# V5 scatter_v2
# ----------------------------------------------------------------------------------------------
def unique_rows(coors, return_counts=False, bounds=None):
    """torch.unique(coors, dim=0, return_inverse=True[, return_counts=True]) for int64 [P,k<=4] rows."""
    _need_cuda(coors)
    assert coors.dtype == torch.int64 and coors.dim() == 2 and coors.shape[1] <= 4
    coors = coors.contiguous()
    P, k = coors.shape
    dev = coors.device
    if P == 0:
        e = coors.new_empty((0,))
        return (coors.clone(), e, e.int()) if return_counts else (coors.clone(), e)
    if bounds is None:
        lo, hi = coors.amin(0).tolist(), coors.amax(0).tolist()
    else:
        lo, hi = bounds
    new_coors = torch.empty((P, k), dtype=torch.int64, device=dev)
    inv = torch.empty((P,), dtype=torch.int64, device=dev)
    cnt = torch.empty((P,), dtype=torch.int32, device=dev) if return_counts else None
    num_dev = torch.empty((1,), dtype=torch.int32, device=dev)
    num_host = C.c_int32(0)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_unique_rows_i64(
        c, coors.data_ptr(), P, k, L.arr(C.c_int64, [int(v) for v in lo]), L.arr(C.c_int64, [int(v) for v in hi]),
        new_coors.data_ptr(), inv.data_ptr(), L.ptr(cnt), num_dev.data_ptr(), C.byref(num_host)))
    M = num_host.value
    if return_counts:
        return new_coors[:M], inv, cnt[:M].long()
    return new_coors[:M], inv


class _SegmentReduce(Function):
    """torch_scatter.scatter / scatter_max, dim=0 (forward + backward)."""

    @staticmethod
    def forward(ctx, src, index, num_segments, mode, want_argmax=True):
        _need_cuda(src, index)
        assert src.dtype == torch.float32 and index.dtype == torch.int64
        src = src.contiguous()
        index = index.contiguous()
        P, Cc = src.shape
        out = torch.empty((num_segments, Cc), dtype=torch.float32, device=src.device)
        arg = torch.empty((num_segments, Cc), dtype=torch.int64, device=src.device) if mode == "max" and want_argmax else None
        c = L.ctx(src.device)
        L.check(c, L.lib().sstb200_segment_reduce(c, src.data_ptr(), index.data_ptr(), P, Cc, num_segments,
                                                  _REDUCE[mode], out.data_ptr(), L.ptr(arg)))
        ctx.mode = mode
        ctx.P = P
        ctx.save_for_backward(index, arg if arg is not None else index)
        if arg is not None:
            ctx.mark_non_differentiable(arg)
            return out, arg
        return out, index.new_empty(0)

    @staticmethod
    def backward(ctx, g, _=None):
        index, arg = ctx.saved_tensors
        g = g.contiguous()
        if ctx.mode == "max":
            gs = g.new_zeros((ctx.P + 1, g.shape[1]))
            gs.scatter_(0, arg, g)
            return gs[:ctx.P], None, None, None, None
        # rows the forward dropped (index outside [0, num_segments)) read the appended zero row
        n = g.shape[0]
        index = torch.where((index >= 0) & (index < n), index, n)
        gv = torch.cat([g, g.new_zeros((1, g.shape[1]))])[index]
        if ctx.mode == "mean":
            cnt = torch.bincount(index, minlength=n + 1).clamp(min=1)
            gv = gv / cnt[index][:, None].to(g.dtype)
        return gv, None, None, None, None


def segment_reduce(src, index, mode, num_segments=None, want_argmax=True):
    """torch_scatter.scatter(src, index, dim=0, reduce=mode) / scatter_max -> (out, argmax or None).  `want_argmax=False`
    skips the argmax output of 'max' (only valid when no gradient is needed): the kernel then runs one FMNMX per element.
    Rows whose index lies outside [0, num_segments) are dropped, forward and backward (their gradient is 0); nothing reports them,
    since that would need a host sync."""
    if num_segments is None:
        num_segments = int(index.max()) + 1 if index.numel() else 0
    if mode == "max" and not want_argmax and src.requires_grad and torch.is_grad_enabled():
        want_argmax = True
    out, arg = _SegmentReduce.apply(src, index, num_segments, mode, want_argmax)
    return out, (arg if mode == "max" and want_argmax else None)


def scatter_v2(feat, coors, mode, return_inv=True, min_points=0, unq_inv=None, new_coors=None):
    """ops/sst/sst_ops.py:151-182."""
    assert feat.size(0) == coors.size(0)
    if mode == "avg":
        mode = "mean"
    if mode not in ("max", "mean", "sum"):
        raise NotImplementedError
    if unq_inv is None:
        new_coors, unq_inv, unq_cnt = unique_rows(coors.long(), return_counts=True)
    else:
        assert new_coors is not None, "please pass new_coors for interface consistency"
    if min_points > 0:
        cnt_per_point = unq_cnt[unq_inv]
        valid_mask = cnt_per_point >= min_points
        feat = feat[valid_mask]
        coors = coors[valid_mask]
        new_coors, unq_inv, unq_cnt = unique_rows(coors.long(), return_counts=True)
    new_feat, _ = segment_reduce(feat, unq_inv, mode, new_coors.shape[0], want_argmax=False)
    if not return_inv:
        return new_feat, new_coors
    return new_feat, new_coors, unq_inv


# ----------------------------------------------------------------------------------------------
# B2 get_inner_win_inds
# ----------------------------------------------------------------------------------------------
class IngroupIndicesFunction(Function):
    """ops/sst/sst_ops.py:244-262."""

    @staticmethod
    def forward(ctx, group_inds):
        _need_cuda(group_inds)
        assert group_inds.dtype == torch.int64 and group_inds.dim() == 1
        group_inds = group_inds.contiguous()
        out_inds = torch.zeros_like(group_inds) - 1
        n = group_inds.numel()
        if n:
            assert int(group_inds.min()) >= 0, "group ids must be non-negative"
            c = L.ctx(group_inds.device)
            L.check(c, L.lib().sstb200_ingroup_indices(c, group_inds.data_ptr(), n, int(group_inds.max()),
                                                       out_inds.data_ptr()))
        ctx.mark_non_differentiable(out_inds)
        return out_inds

    @staticmethod
    def backward(ctx, g):
        return None


get_inner_win_inds = IngroupIndicesFunction.apply


# ----------------------------------------------------------------------------------------------
# B1/B3/B4 fused window plan (one shift)
# ----------------------------------------------------------------------------------------------
class _WindowCfg(C.Structure):
    _fields_ = [("sparse_shape", C.c_int32 * 3), ("window_shape", C.c_int32 * 3), ("batch_size", C.c_int32),
                ("num_levels", C.c_int32), ("level_id", C.c_int32 * 8), ("level_lo", C.c_int32 * 8),
                ("level_hi", C.c_int32 * 8), ("level_max_tokens", C.c_int32 * 8)]


class _WindowShift(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("batch_win_inds", "coors_in_win", "drop_level", "flat2win_inds", "pos_code",
                                          "tok_win", "tok_inner", "win_offsets", "tok_perm", "win_level", "win_rank",
                                          "counters", "tok_slot", "win_batch")]


L.SIGNATURES["sstb200_window_plan"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.POINTER(_WindowCfg), C.c_int, L.vp,
                                                 C.POINTER(_WindowShift), L.P_i32])
L.SIGNATURES["sstb200_window_plan_i32"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.POINTER(_WindowCfg), C.c_int,
                                                     C.POINTER(_WindowShift)])


def _window_shape3(window_shape, sparse_shape):
    if len(window_shape) == 2:
        return (int(window_shape[0]), int(window_shape[1]), int(sparse_shape[-1]))
    return tuple(int(v) for v in window_shape)


def _window_cfg(sparse_shape, window_shape, drop_info, batch_size):
    cfg = _WindowCfg()
    w3 = _window_shape3(window_shape, sparse_shape)
    for i in range(3):
        cfg.sparse_shape[i] = int(sparse_shape[i])
        cfg.window_shape[i] = w3[i]
    cfg.batch_size = int(batch_size)
    keys = list(drop_info.keys())
    assert 1 <= len(keys) <= 8, "at most 8 drop levels supported"
    cfg.num_levels = len(keys)
    for s, k in enumerate(keys):
        lo, hi = drop_info[k]["drop_range"]
        cfg.level_id[s] = int(k)
        cfg.level_lo[s] = int(min(lo, 2 ** 31 - 1))
        cfg.level_hi[s] = int(min(hi, 2 ** 31 - 1))
        cfg.level_max_tokens[s] = int(drop_info[k]["max_tokens"])
    return cfg, keys


class WindowPlan:
    """Device-resident result of sstb200_window_plan for one shift."""
    __slots__ = ("n", "batch_win_inds", "coors_in_win", "drop_level", "flat2win_inds", "pos_code", "tok_win",
                 "tok_inner", "win_offsets", "tok_perm", "win_level", "win_rank", "counters", "tok_slot", "win_batch", "level_keys",
                 "num_windows", "level_windows", "level_tokens", "status")


def window_plan(coors, sparse_shape, window_shape, drop_info, do_shift, batch_size, token_level=None, sync=True):
    """coors [n,4] int64 (b,z,y,x) on CUDA.  Returns a WindowPlan (reference index tensors + window CSR)."""
    _need_cuda(coors)
    assert coors.dtype == torch.int64 and coors.dim() == 2 and coors.shape[1] == 4
    coors = coors.contiguous()
    n, dev = coors.shape[0], coors.device
    cfg, keys = _window_cfg(sparse_shape, window_shape, drop_info, batch_size)
    p = WindowPlan()
    p.n, p.level_keys = n, keys
    i64 = dict(dtype=torch.int64, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    p.batch_win_inds = torch.empty((n,), **i64)
    p.coors_in_win = torch.empty((n, 3), **i64)
    p.drop_level = torch.empty((n,), **i64)
    p.flat2win_inds = torch.empty((n,), **i64)
    p.pos_code = torch.empty((n,), **i32)
    p.tok_win = torch.empty((n,), **i32)
    p.tok_inner = torch.empty((n,), **i32)
    p.win_offsets = torch.empty((n + 1,), **i32)
    p.tok_perm = torch.empty((n,), **i32)
    p.win_level = torch.empty((n,), **i32)
    p.win_rank = torch.empty((n,), **i32)
    p.counters = torch.zeros((20,), **i32)
    p.tok_slot = torch.empty((n,), **i32)
    p.win_batch = torch.empty((n + 16,), **i32)   # int4 records, n/112 + 2 of them
    out = _WindowShift(*[getattr(p, k).data_ptr() for k, _ in _WindowShift._fields_])
    status = (C.c_int32 * 18)()
    if token_level is not None:
        assert token_level.dtype == torch.int64 and token_level.is_cuda and token_level.is_contiguous()
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_window_plan(c, coors.data_ptr(), n, None, C.byref(cfg), int(bool(do_shift)),
                                           L.ptr(token_level), C.byref(out), status if sync else None))
    if sync:
        p.status = status[0]
        if status[0] & 1:
            raise L.SSTB200Error("window_plan: voxel coordinate outside batch_size/sparse_shape window grid")
        if status[0] & 2:
            raise AssertionError("a window's token count is not covered by any drop_range (reference asserts too)")
        p.num_windows = status[1]
        p.level_windows = list(status[2:2 + len(keys)])
        p.level_tokens = list(status[10:10 + len(keys)])
    return p


@torch.no_grad()
def get_window_coors(coors, sparse_shape, window_shape, do_shift):
    """ops/sst/sst_ops.py:266-314."""
    assert sparse_shape[2] < sparse_shape[0], "Usually holds... in case of wrong order"
    n = coors.shape[0]
    if n == 0:
        return coors.new_empty((0,)), coors.new_empty((0, 3))
    B = int(coors[:, 0].max()) + 1
    p = window_plan(coors.long(), sparse_shape, window_shape, {0: dict(max_tokens=1, drop_range=(0, 2 ** 31 - 1))},
                    do_shift, B)
    return p.batch_win_inds, p.coors_in_win


@torch.no_grad()
def make_continuous_inds(inds):
    """ops/sst/sst_ops.py:316-331."""
    if inds.numel() == 0:
        return inds.clone()
    return unique_rows(inds.long().view(-1, 1))[1].to(inds.dtype)


@torch.no_grad()
def get_flat2win_inds(batch_win_inds, voxel_drop_lvl, drop_info, debug=True):
    """ops/sst/sst_ops.py:27-64 (compat path; the fused path is window_plan)."""
    d = {}
    for dl in drop_info:
        dl_mask = voxel_drop_lvl == dl
        if not dl_mask.any():
            continue
        conti = make_continuous_inds(batch_win_inds[dl_mask])
        inner = get_inner_win_inds(conti)
        d[dl] = (conti * drop_info[dl]["max_tokens"] + inner, torch.where(dl_mask))
    return d


def get_flat2win_inds_v2(batch_win_inds, voxel_drop_lvl, drop_info, debug=True):
    d = get_flat2win_inds(batch_win_inds, voxel_drop_lvl, drop_info, debug)
    d["voxel_drop_level"] = voxel_drop_lvl
    d["batching_info"] = drop_info
    return d


def flat2window(feat, voxel_drop_lvl, flat2win_inds_dict, drop_info, padding=0):
    """ops/sst/sst_ops.py:67-104.  Reference-layout (padded [R,T,C]) materialisation: API parity only - the
    attention kernels of this build consume the ragged CSR and never call this."""
    out = {}
    for dl in drop_info:
        dl_mask = voxel_drop_lvl == dl
        if not dl_mask.any():
            continue
        this_inds = flat2win_inds_dict[dl][0]
        T = drop_info[dl]["max_tokens"]
        R = int((this_inds // T).max()) + 1
        buf = torch.full((R * T, feat.shape[-1]), padding, dtype=feat.dtype, device=feat.device)
        buf[this_inds] = feat[dl_mask]
        out[dl] = buf.reshape(R, T, feat.shape[-1])
    return out


def window2flat(feat_3d_dict, inds_dict):
    """ops/sst/sst_ops.py:106-132."""
    n = sum(inds_dict[dl][0].shape[0] for dl in inds_dict)
    first = feat_3d_dict[next(iter(feat_3d_dict))]
    out = torch.zeros((n, first.shape[-1]), device=first.device, dtype=first.dtype)
    for dl in feat_3d_dict:
        inds, flat_pos = inds_dict[dl]
        out[flat_pos] = feat_3d_dict[dl].reshape(-1, first.shape[-1])[inds]
    return out


def window2flat_v2(feat_3d_dict, inds_dict):
    return window2flat(feat_3d_dict, {k: inds_dict[k] for k in inds_dict if not isinstance(k, str)})


def flat2window_v2(feat, inds_dict, padding=0):
    assert "voxel_drop_level" in inds_dict, "voxel_drop_level should be in inds_dict in v2 function"
    inds_v1 = {k: inds_dict[k] for k in inds_dict if not isinstance(k, str)}
    return flat2window(feat, inds_dict["voxel_drop_level"], inds_v1, inds_dict["batching_info"], padding=padding)


# ----------------------------------------------------------------------------------------------
# S3 small builders (host logic only)
# ----------------------------------------------------------------------------------------------
def get_activation(activation):
    """ops/sst/sst_ops.py:363-371."""
    if activation == "relu":
        return torch.nn.functional.relu
    if activation == "gelu":
        return torch.nn.functional.gelu
    if activation == "glu":
        return torch.nn.functional.glu
    raise RuntimeError(f"activation should be relu/gelu, not {activation}.")


def get_activation_layer(act, dim=None):
    """ops/sst/sst_ops.py:373-392."""
    act = act.lower()
    table = {"relu": lambda: nn.ReLU(inplace=True), "gelu": nn.GELU, "leakyrelu": lambda: nn.LeakyReLU(inplace=True),
             "prelu": lambda: nn.PReLU(num_parameters=dim), "swish": lambda: nn.SiLU(inplace=True),
             "silu": lambda: nn.SiLU(inplace=True), "glu": nn.GLU, "elu": lambda: nn.ELU(inplace=True)}
    if act not in table:
        raise NotImplementedError
    return table[act]()


def build_norm_layer(cfg, num_features):
    """mmcv.cnn.build_norm_layer for the norm types the path uses; returns (name, layer)."""
    from .norm import NaiveSyncBatchNorm1d, NaiveSyncBatchNorm2d
    cfg = dict(cfg)
    t = cfg.pop("type")
    cfg.pop("requires_grad", None)
    if t == "LN":
        return "ln", nn.LayerNorm(num_features, **cfg)
    if t in ("BN1d", "BN"):
        return "bn", nn.BatchNorm1d(num_features, **cfg)
    if t == "naiveSyncBN1d":
        return "bn", NaiveSyncBatchNorm1d(num_features, **cfg)
    if t == "BN2d":
        return "bn", nn.BatchNorm2d(num_features, **cfg)
    if t == "naiveSyncBN2d":
        return "bn", NaiveSyncBatchNorm2d(num_features, **cfg)
    raise NotImplementedError(f"norm type {t}")


def build_mlp(in_channel, hidden_dims, norm_cfg, is_head=False, act="relu", bias=False, dropout=0):
    """ops/sst/sst_ops.py:334-361 (parameter container: `mlp.{i}.0.weight`, `mlp.{i}.1.{weight,bias}`)."""
    layers = []
    last = in_channel
    if isinstance(hidden_dims, int):
        hidden_dims = [hidden_dims]
    for i, ch in enumerate(hidden_dims):
        if i == len(hidden_dims) - 1 and is_head:
            layers.append(nn.Linear(last, ch, bias=True))
        else:
            sq = [nn.Linear(last, ch, bias=bias), build_norm_layer(norm_cfg, ch)[1], get_activation_layer(act, ch)]
            if dropout > 0:
                sq.append(nn.Dropout(dropout))
            layers.append(nn.Sequential(*sq))
        last = ch
    return nn.Sequential(*layers)


L.SIGNATURES["sstb200_linear"] = (C.c_int, [L.vp, L.vp, L.vp, L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int])


def linear(x, weight, bias=None, act=None):
    """nn.Linear forward (fp32) through libsstb200; act in (None, 'relu', 'gelu')."""
    _need_cuda(x, weight)
    x = x.float().contiguous()
    w = weight.detach().float().contiguous()
    b = None if bias is None else bias.detach().float().contiguous()
    out = torch.empty((x.shape[0], w.shape[0]), dtype=torch.float32, device=x.device)
    c = L.ctx(x.device)
    L.check(c, L.lib().sstb200_linear(c, x.data_ptr(), w.data_ptr(), L.ptr(b), out.data_ptr(), x.shape[0], w.shape[0],
                                      w.shape[1], {None: 0, "relu": 1, "gelu": 2}[act]))
    return out


# ----------------------------------------------------------------------------------------------
# FSD RoI point pooling (ops/dynamic_point_pool_op.py:9-113)
# ----------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_dynamic_point_pool"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, L.vp, L.vp, C.c_int, L.P_f32, C.c_int, C.c_int,
                                                        C.c_int, L.vp, L.vp, L.vp, L.vp, L.P_i32])


def point_pool(rois, rois_batch, pts, pts_batch, extra_wlh, max_inbox_point, max_all_pts, per_sample=False, num_samples=1):
    """sstb200_dynamic_point_pool -> (pts_idx int64 [K], roi_idx int64 [K], feats fp32 [K, 13]).  per_sample: max_all_pts and the fake
    row apply to every sample (RoIs grouped by ascending batch id, num_samples distinct ids) instead of to the whole call."""
    _need_cuda(rois, pts, rois_batch, pts_batch)
    rois = rois.float().contiguous()
    pts = pts[:, :3].float().contiguous()
    rb = None if rois_batch is None else rois_batch.int().contiguous()
    pb = None if pts_batch is None else pts_batch.int().contiguous()
    cap = int(max_all_pts) * (int(num_samples) if per_sample else 1)
    dev = pts.device
    out_idx = torch.empty((cap,), dtype=torch.int64, device=dev)
    out_roi = torch.empty((cap,), dtype=torch.int64, device=dev)
    out_feats = torch.empty((cap, 13), dtype=torch.float32, device=dev)
    num_dev = torch.empty((1,), dtype=torch.int32, device=dev)
    num_host = (C.c_int32 * 3)()
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_dynamic_point_pool(c, rois.data_ptr(), L.ptr(rb), rois.shape[0], pts.data_ptr(), L.ptr(pb), pts.shape[0],
                                                  L.arr(C.c_float, [float(v) for v in extra_wlh]), int(max_inbox_point), int(max_all_pts),
                                                  int(bool(per_sample)), out_idx.data_ptr(), out_roi.data_ptr(), out_feats.data_ptr(),
                                                  num_dev.data_ptr(), num_host))
    k, found, written = num_host[0], num_host[1], num_host[2]
    if found > written:
        import warnings
        warnings.warn(f"dynamic_point_pool: {found - written} of {found} RoI-point pairs exceed max_all_pts={max_all_pts} and were dropped")
    return out_idx[:k], out_roi[:k], out_feats[:k]


class DynamicPointPoolFunction(Function):
    """dynamic_point_pool_op.py:9-58.  rois [R, 7] (x, y, z_bottom, w, l, h, rz), pts [N, 3] -> point index, RoI index, features
    [K, 13] = point xyz, local xyz, 6 boundary offsets, is_in_margin; rows sorted by RoI then point index; one (-1, -1, 0) row when no
    point lies in any enlarged box.  Deterministic."""

    @staticmethod
    def forward(ctx, rois, pts, extra_wlh, max_inbox_point, max_all_pts=50000):
        assert len(rois) > 0
        out = point_pool(rois, None, pts, None, extra_wlh, max_inbox_point, max_all_pts)
        for t in out:
            ctx.mark_non_differentiable(t)
        return out

    @staticmethod
    def backward(ctx, g1, g2, g3):
        return None, None, None, None, None


dynamic_point_pool = DynamicPointPoolFunction.apply


class DynamicPointPoolMixedFunction(Function):
    """dynamic_point_pool_op.py:63-111: as above over several samples at once; a point pairs only with RoIs of its own batch id."""

    @staticmethod
    def forward(ctx, rois, rois_batch, pts, pts_batch, extra_wlh, max_inbox_point, max_all_pts=200000):
        assert len(rois) > 0
        out = point_pool(rois, rois_batch, pts, pts_batch, extra_wlh, max_inbox_point, max_all_pts)
        for t in out:
            ctx.mark_non_differentiable(t)
        return out

    @staticmethod
    def backward(ctx, g1, g2, g3):
        return None, None, None, None, None, None, None


dynamic_point_pool_mixed = DynamicPointPoolMixedFunction.apply


# ----------------------------------------------------------------------------------------------
# Rotated BEV overlap / IoU / NMS (ops/iou3d/iou3d_utils.py, core/post_processing/box3d_nms.py:10-143)
# ----------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_boxes_overlap_bev"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.c_int, L.vp])
L.SIGNATURES["sstb200_boxes_iou_bev"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.c_int, L.vp])
L.SIGNATURES["sstb200_nms_bev_workspace_bytes"] = (C.c_int, [L.vp, C.c_int, L.P_i32, C.c_int, L.P_i64])
L.SIGNATURES["sstb200_nms_bev"] = (C.c_int, [L.vp, L.vp, C.c_int, L.P_i32, C.c_int, L.P_f32, C.c_int, L.vp, C.c_int64, L.vp, L.vp,
                                             L.P_i32])


def _bev_boxes(boxes, name):
    if boxes.dim() != 2 or boxes.shape[1] != 5:
        raise L.SSTB200Error(f"{name}: boxes must be [N, 5] (x1, y1, x2, y2, r), got {tuple(boxes.shape)}")
    return boxes.float().contiguous()


def _bev_pairs(fn, boxes_a, boxes_b):
    _need_cuda(boxes_a, boxes_b)
    a, b = _bev_boxes(boxes_a, fn), _bev_boxes(boxes_b, fn)
    out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    c = L.ctx(a.device)
    L.check(c, getattr(L.lib(), fn)(c, a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], out.data_ptr()))
    return out


def boxes_iou_bev(boxes_a, boxes_b):
    """iou3d_utils.py:12-28: rotated BEV IoU of boxes_a [M, 5] and boxes_b [N, 5] ([x1, y1, x2, y2, r]) -> fp32 [M, N]."""
    return _bev_pairs("sstb200_boxes_iou_bev", boxes_a, boxes_b)


def boxes_overlap_bev(boxes_a, boxes_b):
    """iou3d_cuda.boxes_overlap_bev_gpu (BaseInstance3DBoxes.overlaps): rotated BEV overlap area, fp32 [M, N]."""
    return _bev_pairs("sstb200_boxes_overlap_bev", boxes_a, boxes_b)


def nms_bev(boxes, seg_offsets, thresh, rotated=True):
    """Segmented greedy NMS (sstb200_nms_bev): boxes [num, 5] grouped into segments [seg_offsets[s], seg_offsets[s+1]), each sorted by
    descending score; thresh[s] per segment (None keeps the whole segment).  Returns int64 positions into `boxes` of the kept boxes,
    segment after segment, in score order; one host sync for their number."""
    keep, num_dev = _nms_bev_async(boxes, seg_offsets, thresh, rotated)
    return keep[:int(num_dev.item())]


def _nms_bev_async(boxes, seg_offsets, thresh, rotated):
    """nms_bev without reading the kept count: (keep int64 [num], whose first num_dev entries are valid, num_dev int32 [1] on the
    device).  No host sync."""
    _need_cuda(boxes)
    b = _bev_boxes(boxes, "nms_bev")
    S = len(seg_offsets) - 1
    off = L.arr(C.c_int32, [int(v) for v in seg_offsets])
    th = L.arr(C.c_float, [math.inf if t is None else float(t) for t in thresh])
    if len(th) != S:
        raise L.SSTB200Error(f"nms_bev: {len(th)} thresholds for {S} segments")
    c = L.ctx(b.device)
    nbytes = C.c_int64()
    L.check(c, L.lib().sstb200_nms_bev_workspace_bytes(c, b.shape[0], off, S, C.byref(nbytes)))
    ws = torch.empty((nbytes.value,), dtype=torch.uint8, device=b.device)
    keep = torch.empty((b.shape[0],), dtype=torch.int64, device=b.device)
    num_dev = torch.empty((1,), dtype=torch.int32, device=b.device)
    L.check(c, L.lib().sstb200_nms_bev(c, b.data_ptr(), b.shape[0], off, S, th, int(bool(rotated)), ws.data_ptr(), nbytes.value,
                                       keep.data_ptr(), num_dev.data_ptr(), None))
    return keep, num_dev


def nms_gpu(boxes, scores, thresh, pre_maxsize=None, post_max_size=None):
    """iou3d_utils.py:31-56: rotated NMS.  boxes [N, 5], scores [N] -> int64 indices into the input of the kept boxes, by descending
    score (the reference's `scores.sort(0, descending=True)`, so ties fall in torch's order as there)."""
    _need_cuda(boxes, scores)
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    keep = order[nms_bev(boxes[order], [0, order.numel()], [thresh], rotated=True)].contiguous()
    if post_max_size is not None:
        keep = keep[:post_max_size]
    return keep


def nms_normal_gpu(boxes, scores, thresh):
    """iou3d_utils.py:106-124: NMS with the axis-aligned IoU (r ignored)."""
    _need_cuda(boxes, scores)
    order = scores.sort(0, descending=True)[1]
    return order[nms_bev(boxes[order], [0, order.numel()], [thresh], rotated=False)].contiguous()


def multiclass_nms_groups(mlvl_bboxes, mlvl_bboxes_for_nms, cls, idx, sc, group, num_groups, num_classes, nms_thrs, max_num, rotated,
                          extras=()):
    """box3d_multiclass_nms (box3d_nms.py:10-143) for `num_groups` independent groups of candidates in ONE segmented nms_bev call.
    Candidate k is box idx[k] of mlvl_bboxes / mlvl_bboxes_for_nms, of class cls[k] in [0, num_classes), with score sc[k], in group
    group[k] (int64 device tensors; group num_groups drops the candidate); within a (group, class) the candidates come in input order.
    nms_thrs: one threshold per class,
    None for no NMS.  Per group, the reference's order: classes in turn; within a class, descending score, or input order for a class
    whose threshold is None; then, over max_num kept, the reference's own `scores.sort(descending=True)` cut.  Returns a list over
    groups of (bboxes, scores, labels, *extras[idx of the kept]) or None for a group with nothing kept.  Whatever the number of groups,
    one host sync for the candidates per (group, class) and, when some class has an NMS threshold, a second for the kept boxes per
    group; with no threshold every candidate is kept and nms_bev is not called."""
    _need_cuda(mlvl_bboxes, mlvl_bboxes_for_nms, cls, idx, sc, group, *extras)
    dev = sc.device
    seg = group * num_classes + cls
    none = [t is None for t in nms_thrs]
    if all(none):                                                      # a class without NMS keeps input order
        key = torch.zeros_like(sc)
    elif any(none):
        key = torch.where(torch.tensor(none, dtype=torch.bool, device=dev)[cls], torch.zeros_like(sc), sc)
    else:
        key = sc
    o = torch.sort(key, descending=True, stable=True).indices
    o = o[torch.sort(seg[o], stable=True).indices]
    S = (num_groups + 1) * num_classes
    counts = torch.zeros((S,), dtype=torch.int64, device=dev).index_add_(0, seg, torch.ones_like(seg))
    counts = counts.tolist()[:num_groups * num_classes]
    n = sum(counts)
    if n == 0:
        return [None] * num_groups
    o = o[:n]                                                          # the dropped candidates sort last
    cls, idx, sc, group = cls[o], idx[o], sc[o], group[o]
    if all(none):                  # nothing to suppress: every candidate is kept, in the order above, and the counts are known
        keep = torch.arange(n, device=dev)
        per = [sum(counts[g * num_classes:(g + 1) * num_classes]) for g in range(num_groups)]
    else:
        keep, num_dev = _nms_bev_async(mlvl_bboxes_for_nms[idx], _offsets(counts), list(nms_thrs) * num_groups, rotated)
        K = keep.shape[0]
        live = torch.arange(K, device=dev) < num_dev
        keep = torch.where(live, keep, torch.zeros_like(keep))
        kept_group = torch.where(live, group[keep], torch.full_like(keep, num_groups))
        per = torch.zeros((num_groups + 1,), dtype=torch.int64, device=dev).index_add_(0, kept_group, torch.ones_like(kept_group))
        per = per.tolist()[:num_groups]
    out = []
    for g, (a, b) in enumerate(zip(_offsets(per), _offsets(per)[1:])):
        if a == b:
            out.append(None)
            continue
        k = keep[a:b]
        sel = idx[k]
        res = [mlvl_bboxes[sel], sc[k], cls[k]] + [e[sel] for e in extras]
        if b - a > max_num:
            _, inds = res[1].sort(descending=True)
            inds = inds[:max_num]
            res = [r[inds] for r in res]
        out.append(tuple(res))
    return out


def box3d_multiclass_nms(mlvl_bboxes, mlvl_bboxes_for_nms, mlvl_scores, score_thr, max_num, cfg, mlvl_dir_scores=None,
                         mlvl_attr_scores=None, mlvl_bboxes2d=None):
    """box3d_nms.py:10-143 with every class in ONE segmented NMS call (the one-group case of multiclass_nms_groups).  Same arguments,
    outputs and order: classes in turn, each class's kept boxes by descending score (boxes in input order for a class whose nms_thr is
    None), then the reference's own `scores.sort(descending=True)` when more than max_num remain.  Within a class, equal scores are
    taken in input order; the reference takes them in torch's sort order, so the two agree whenever a class has no tied scores."""
    _need_cuda(mlvl_bboxes, mlvl_bboxes_for_nms, mlvl_scores, mlvl_dir_scores, mlvl_attr_scores, mlvl_bboxes2d)
    num_classes = mlvl_scores.shape[1] - 1
    dev = mlvl_scores.device
    if isinstance(score_thr, (list, tuple)):
        assert len(score_thr) == num_classes
        score_thrs = list(score_thr)
    else:
        score_thrs = [score_thr] * num_classes
    nms_thr = cfg.nms_thr
    if isinstance(nms_thr, (list, tuple)):
        assert len(nms_thr) == num_classes
        nms_thrs = list(nms_thr)
    else:
        nms_thrs = [nms_thr] * num_classes
    cls_scores = mlvl_scores[:, :num_classes]
    thr = torch.tensor([float(t) for t in score_thrs], dtype=mlvl_scores.dtype, device=dev)
    cls, idx = (cls_scores > thr).t().nonzero(as_tuple=True)           # class-major, input order within a class
    given = [e for e in (mlvl_dir_scores, mlvl_attr_scores, mlvl_bboxes2d) if e is not None]
    res = multiclass_nms_groups(mlvl_bboxes, mlvl_bboxes_for_nms, cls, idx, cls_scores[idx, cls], torch.zeros_like(cls), 1,
                                num_classes, nms_thrs, max_num, cfg.use_rotate_nms, given)[0]
    if res is None:
        res = (mlvl_scores.new_zeros((0, mlvl_bboxes.size(-1))), mlvl_scores.new_zeros((0,)), mlvl_scores.new_zeros((0,), dtype=torch.long))
        res = res + tuple(mlvl_scores.new_zeros((0, 4) if e is mlvl_bboxes2d else (0,)) for e in given)
    return res


# ----------------------------------------------------------------------------------------------
# Points in boxes and RoI-aware pooling (ops/roiaware_pool3d: points_in_boxes.py, roiaware_pool3d.py)
# ----------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_points_in_boxes"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int, L.vp])
L.SIGNATURES["sstb200_roiaware_pool3d_plan"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, L.vp, L.vp, C.c_int, L.P_i32, C.c_int, L.P_i64])
L.SIGNATURES["sstb200_roiaware_pool3d_forward"] = (C.c_int, [L.vp, L.vp, C.c_int, C.c_int, L.vp, L.vp, L.vp, L.vp, L.vp, L.vp])
L.SIGNATURES["sstb200_roiaware_pool3d_backward"] = (C.c_int, [L.vp, C.c_int, C.c_int, C.c_int, C.c_int64, L.vp, L.vp, L.vp, L.vp, L.vp,
                                                              L.vp, L.vp])


def _points_in_boxes(points, boxes, mode):
    assert boxes.shape[0] == points.shape[0], \
        f'Points and boxes should have the same batch size, got {boxes.shape[0]} and {points.shape[0]}'
    assert boxes.shape[2] == 7, f'boxes dimension should be 7, got unexpected shape {boxes.shape[2]}'
    assert points.shape[2] == 3, f'points dimension should be 3, got unexpected shape {points.shape[2]}'
    _need_cuda(points, boxes)
    assert points.device == boxes.device, 'Points and boxes should be put on the same device'
    B, M, _ = points.shape
    T = boxes.shape[1]
    out = torch.empty((B, M) if mode == 0 else (B, M, T), dtype=torch.int32, device=points.device)
    p, b = points.float().contiguous(), boxes.float().contiguous()
    c = L.ctx(points.device)
    L.check(c, L.lib().sstb200_points_in_boxes(c, p.data_ptr(), b.data_ptr(), B, M, T, mode, out.data_ptr()))
    return out


def points_in_boxes_gpu(points, boxes):
    """points_in_boxes.py:6-47: points [B, M, 3], boxes [B, T, 7] (x, y, z_bottom, w, l, h, rz) -> int32 [B, M], the lowest index of a
    box holding the point, -1 for none (overlapping boxes: the first one wins, as in the reference's loop)."""
    return _points_in_boxes(points, boxes, 0)


def points_in_boxes_batch(points, boxes):
    """points_in_boxes.py:85-123: points [B, M, 3], boxes [B, T, 7] -> int32 [B, M, T], 1 where the point is inside the box, else 0."""
    return _points_in_boxes(points, boxes, 1)


_POOL3D_MODES = {"max": 0, "avg": 1}


def _out_size3(out_size):
    if isinstance(out_size, int):
        return (out_size,) * 3
    assert len(out_size) == 3 and all(isinstance(v, int) for v in out_size), f"out_size must be an int or 3 ints, got {out_size!r}"
    return tuple(out_size)


def roiaware_pool3d_forward(rois, pts, pts_feature, out_size, max_pts_per_voxel, mode, rois_batch=None, pts_batch=None):
    """sstb200_roiaware_pool3d_plan + _forward.  rois [R, 7], pts [N, 3], pts_feature [N, C]; mode 0 (max) or 1 (avg); optional int32
    batch ids of RoIs and points (a point pairs only with RoIs of its own batch id).  Returns pooled [R, ox, oy, oz, C] and the compact
    state of the backward: (voxel_slot, voxel_offsets, point_idx, argmax or None, counts, num_pairs).  One stream sync."""
    if mode not in (0, 1):
        raise L.SSTB200Error(f"roiaware_pool3d: mode must be 0 (max) or 1 (avg), got {mode!r}")
    ox, oy, oz = _out_size3(out_size)
    if not all(1 <= v <= 255 for v in (ox, oy, oz)):      # the reference asserts < 256 (voxel indices are packed into 8 bits each)
        raise L.SSTB200Error(f"roiaware_pool3d: out_size {(ox, oy, oz)} outside [1, 255]")
    if int(max_pts_per_voxel) < 1:
        raise L.SSTB200Error(f"roiaware_pool3d: max_pts_per_voxel must be >= 1, got {max_pts_per_voxel}")
    _need_cuda(rois, pts, pts_feature, rois_batch, pts_batch)
    rois, pts, feats = rois.float().contiguous(), pts.float().contiguous(), pts_feature.float().contiguous()
    assert rois.dim() == 2 and rois.shape[1] == 7 and pts.dim() == 2 and pts.shape[1] == 3
    assert feats.dim() == 2 and feats.shape[0] == pts.shape[0]
    rb = None if rois_batch is None else rois_batch.int().contiguous()
    pb = None if pts_batch is None else pts_batch.int().contiguous()
    R, N, Ch = rois.shape[0], pts.shape[0], feats.shape[1]
    dev = pts.device
    c = L.ctx(dev)
    P = C.c_int64()
    L.check(c, L.lib().sstb200_roiaware_pool3d_plan(c, rois.data_ptr(), L.ptr(rb), R, pts.data_ptr(), L.ptr(pb), N,
                                                    L.arr(C.c_int32, [ox, oy, oz]), int(max_pts_per_voxel), C.byref(P)))
    P = P.value
    pooled = torch.empty((R, ox, oy, oz, Ch), dtype=torch.float32, device=dev)
    slot = torch.empty((max(P, 1),), dtype=torch.int64, device=dev)
    voff = torch.empty((P + 1,), dtype=torch.int32, device=dev)
    pidx = torch.empty((max(P, 1),), dtype=torch.int32, device=dev)
    argmax = torch.empty((max(P, 1), Ch), dtype=torch.int32, device=dev) if mode == 0 else None
    counts = torch.empty((2,), dtype=torch.int32, device=dev)
    L.check(c, L.lib().sstb200_roiaware_pool3d_forward(c, feats.data_ptr(), Ch, mode, pooled.data_ptr(), slot.data_ptr(), voff.data_ptr(),
                                                       pidx.data_ptr(), L.ptr(argmax), counts.data_ptr()))
    return pooled, (slot, voff, pidx, argmax, counts, P)


def roiaware_pool3d_backward(grad_out, state, num_pts, mode):
    """sstb200_roiaware_pool3d_backward: grad_out [R, ox, oy, oz, C] -> grad_in [num_pts, C] (bit-identical from run to run)."""
    slot, voff, pidx, argmax, counts, P = state
    g = grad_out.float().contiguous()
    Ch = g.shape[-1]
    grad_in = torch.empty((num_pts, Ch), dtype=torch.float32, device=g.device)
    c = L.ctx(g.device)
    L.check(c, L.lib().sstb200_roiaware_pool3d_backward(c, num_pts, Ch, mode, P, slot.data_ptr(), voff.data_ptr(), pidx.data_ptr(),
                                                        L.ptr(argmax), counts.data_ptr(), g.data_ptr(), grad_in.data_ptr()))
    return grad_in


class RoIAwarePool3dFunction(Function):
    """roiaware_pool3d.py:45-86: rois [R, 7] (x, y, z_bottom, w, l, h, rz), pts [N, 3], pts_feature [N, C], out_size (int or 3 ints),
    max_pts_per_voxel m, mode 0 (max) / 1 (avg) -> pooled [R, ox, oy, oz, C]; gradient for pts_feature only.  The saved state is compact
    (occupied voxels, their kept points, [occupied, C] argmax) instead of the reference's dense [R, ox, oy, oz, m] index buffer.
    Optional rois_batch / pts_batch pool every sample of a batch in one call."""

    @staticmethod
    def forward(ctx, rois, pts, pts_feature, out_size, max_pts_per_voxel, mode, rois_batch=None, pts_batch=None):
        pooled, state = roiaware_pool3d_forward(rois, pts, pts_feature, out_size, max_pts_per_voxel, mode, rois_batch, pts_batch)
        ctx.roiaware_pool3d_for_backward = (state, mode, pts.shape[0])
        return pooled

    @staticmethod
    def backward(ctx, grad_out):
        state, mode, num_pts = ctx.roiaware_pool3d_for_backward
        return None, None, roiaware_pool3d_backward(grad_out, state, num_pts, mode), None, None, None, None, None


class RoIAwarePool3d(nn.Module):
    """roiaware_pool3d.py:8-42: RoIAwarePool3d(out_size, max_pts_per_voxel=128, mode='max'); forward(rois, pts, pts_feature)."""

    def __init__(self, out_size, max_pts_per_voxel=128, mode='max'):
        super().__init__()
        self.out_size = out_size
        self.max_pts_per_voxel = max_pts_per_voxel
        assert mode in ['max', 'avg']
        self.mode = _POOL3D_MODES[mode]

    def forward(self, rois, pts, pts_feature):
        return RoIAwarePool3dFunction.apply(rois, pts, pts_feature, self.out_size, self.max_pts_per_voxel, self.mode)


# ----------------------------------------------------------------------------------------------
# deformable convolution (mmcv.ops.deform_conv 1.3.8-1.4.0: deform_conv2d / DeformConv2dFunction)
# ----------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_dcn_forward"] = (C.c_int, [L.vp, L.P_i32, L.vp, L.vp, L.vp, L.vp])
L.SIGNATURES["sstb200_dcn_backward_workspace_bytes"] = (C.c_int, [L.vp, L.P_i32, L.P_i64])
L.SIGNATURES["sstb200_dcn_backward"] = (C.c_int, [L.vp, L.P_i32, L.vp, L.vp, L.vp, L.vp, L.vp, C.c_int64, L.vp, L.vp, L.vp])


def _dcn_pair(v, name):
    v = (v, v) if isinstance(v, int) else tuple(v)
    if len(v) != 2 or not all(isinstance(i, int) for i in v):
        raise L.SSTB200Error(f"deform_conv2d: {name} must be an int or a pair of ints, got {v!r}")
    return v


def _dcn_geom(input, offset, weight, stride, padding, dilation, groups, deform_groups):
    """validated geom[15] of the C ABI for fp32 CUDA tensors of mmcv's shapes"""
    for name, t in (("input", input), ("offset", offset), ("weight", weight)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 4:
            raise L.SSTB200Error(f"deform_conv2d: {name} must be a 4-d float32 CUDA tensor (there is no CPU or fp16 path)")
    (sh, sw), (ph, pw), (dh, dw) = _dcn_pair(stride, "stride"), _dcn_pair(padding, "padding"), _dcn_pair(dilation, "dilation")
    N, Cin, H, W = input.shape
    Cout, cg, kh, kw = weight.shape
    if groups < 1 or deform_groups < 1 or Cin != cg * groups or Cout % groups or Cin % deform_groups:
        raise L.SSTB200Error(f"deform_conv2d: input {tuple(input.shape)} / weight {tuple(weight.shape)} do not fit groups {groups} and "
                             f"deform_groups {deform_groups}")
    if min(sh, sw, dh, dw) < 1 or min(ph, pw) < 0:
        raise L.SSTB200Error("deform_conv2d: stride and dilation must be >= 1, padding >= 0")
    Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
    Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    if Ho < 1 or Wo < 1 or tuple(offset.shape) != (N, 2 * deform_groups * kh * kw, Ho, Wo):
        raise L.SSTB200Error(f"deform_conv2d: offset {tuple(offset.shape)} is not [N, 2 * deform_groups * kh * kw, Ho, Wo] = "
                             f"{(N, 2 * deform_groups * kh * kw, Ho, Wo)}")
    if not (input.device == offset.device == weight.device):
        raise L.SSTB200Error("deform_conv2d: input, offset and weight must be on one device")
    return L.arr(C.c_int32, [N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, groups, deform_groups]), (N, Cout, Ho, Wo)


class DeformConv2dFunction(Function):
    """mmcv's DeformConv2dFunction.apply(input, offset, weight, stride, padding, dilation, groups, deform_groups, bias, im2col_step).
    Backward re-samples (nothing beyond the inputs is saved) and is deterministic: no float atomics."""

    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False, im2col_step=32):
        if bias:
            raise L.SSTB200Error("deform_conv2d: bias=True is not supported (as in mmcv's DeformConv2d)")
        geom, out_shape = _dcn_geom(input, offset, weight, stride, padding, dilation, groups, deform_groups)
        x, off, w = input.contiguous(), offset.contiguous(), weight.contiguous()
        y = torch.empty(out_shape, dtype=torch.float32, device=x.device)
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_dcn_forward(c, geom, L.ptr(x), L.ptr(off), L.ptr(w), L.ptr(y)))
        ctx.save_for_backward(x, off, w)
        ctx.geom = list(geom)
        return y

    @staticmethod
    def backward(ctx, grad_y):
        x, off, w = ctx.saved_tensors
        gx, goff, gw = deform_conv2d_backward(x, off, w, grad_y, ctx.geom, *ctx.needs_input_grad[:3])
        return gx, goff, gw, None, None, None, None, None, None, None


def deform_conv2d_backward(x, offset, weight, grad_y, geom, want_x=True, want_offset=True, want_weight=True):
    """(grad_x, grad_offset, grad_weight); a gradient not wanted is None and is not computed"""
    geom = L.arr(C.c_int32, list(geom))
    gy = grad_y.contiguous()
    gx = torch.empty_like(x) if want_x else None
    goff = torch.empty_like(offset) if want_offset else None
    gw = torch.empty_like(weight) if want_weight else None
    if not (want_x or want_offset or want_weight):
        return gx, goff, gw
    c = L.ctx(x.device)
    nbytes = C.c_int64()
    L.check(c, L.lib().sstb200_dcn_backward_workspace_bytes(c, geom, C.byref(nbytes)))
    ws = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=x.device)
    L.check(c, L.lib().sstb200_dcn_backward(c, geom, L.ptr(x), L.ptr(offset), L.ptr(weight), L.ptr(gy), L.ptr(ws), nbytes.value,
                                            L.ptr(gx), L.ptr(goff), L.ptr(gw)))
    return gx, goff, gw


def deform_conv2d_workspace_bytes(input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deform_groups=1):
    """device bytes the backward of this call borrows (caller-owned workspace of sstb200_dcn_backward)"""
    geom, _ = _dcn_geom(input, offset, weight, stride, padding, dilation, groups, deform_groups)
    c = L.ctx(input.device)
    nbytes = C.c_int64()
    L.check(c, L.lib().sstb200_dcn_backward_workspace_bytes(c, geom, C.byref(nbytes)))
    return nbytes.value


def deform_conv2d(input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False, im2col_step=32):
    """mmcv.ops.deform_conv2d: fp32 NCHW input [N, Cin, H, W], offset [N, 2 dg kh kw, Ho, Wo], weight [Cout, Cin / groups, kh, kw] ->
    [N, Cout, Ho, Wo].  im2col_step is accepted and ignored (one launch covers the batch)."""
    return DeformConv2dFunction.apply(input, offset, weight, stride, padding, dilation, groups, deform_groups, bias, im2col_step)


# ----------------------------------------------------------------------------------------------
# CenterHead training (mmdet3d/models/dense_heads/centerpoint_head.py:421-610)
# ----------------------------------------------------------------------------------------------
_PP = C.POINTER(C.c_void_p)
L.SIGNATURES["sstb200_centerpoint_targets"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int, L.P_i32, C.c_int, L.P_i32, C.c_int, L.P_f32, L.P_f32,
                                                         C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, _PP, _PP, _PP,
                                                         _PP])
L.SIGNATURES["sstb200_gaussian_focal_loss_forward"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int64, C.c_float, L.vp, L.vp])
L.SIGNATURES["sstb200_gaussian_focal_loss_backward"] = (C.c_int, [L.vp, L.vp, L.vp, C.c_int64, C.c_float, L.vp, L.vp, L.vp])
L.SIGNATURES["sstb200_centerpoint_l1_loss_forward"] = (C.c_int, [L.vp, _PP, C.c_int, C.c_int, C.c_int, L.vp, L.vp, L.vp, C.c_int, L.P_f32,
                                                                 C.c_float, L.vp])
L.SIGNATURES["sstb200_centerpoint_l1_loss_backward"] = (C.c_int, [L.vp, _PP, C.c_int, C.c_int, C.c_int, L.vp, L.vp, L.vp, C.c_int, L.P_f32,
                                                                  C.c_float, L.vp, _PP])

CENTERPOINT_HEADS = (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _fp32_cuda(name, t, dim=None):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise L.SSTB200Error(f"{name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype == torch.float16:                       # @force_fp32 casts half predictions
        t = t.float()
    if t.dtype != torch.float32:
        raise L.SSTB200Error(f"{name} must be float32, got {t.dtype}")
    if dim is not None and t.dim() != dim:
        raise L.SSTB200Error(f"{name} must be {dim}-d, got shape {tuple(t.shape)}")
    return t.contiguous()


def _offsets(sizes):
    out = [0]
    for n in sizes:
        out.append(out[-1] + int(n))
    return out


def _sample_offsets(fn, sample_sizes, n):
    sizes = [int(v) for v in sample_sizes]
    if sum(sizes) != n or min(sizes, default=-1) < 0:
        raise L.SSTB200Error(f"{fn}: sample sizes {sizes} do not add up to the {n} boxes")
    return _offsets(sizes)


def _cat_gt(fn, gt_boxes, gt_labels, dev):
    """per-sample boxes (columns 0-6 of tensors or of their `.tensor`) and labels -> fp32 [G, 7], int64 [G] on dev, B + 1 offsets"""
    boxes = [getattr(b, "tensor", b) for b in gt_boxes]
    for b, lab in zip(boxes, gt_labels):
        if b.dim() != 2 or b.shape[1] < 7 or lab.shape != (b.shape[0],):
            raise L.SSTB200Error(f"{fn}: boxes {tuple(b.shape)} and labels {tuple(lab.shape)} do not match")
    gt = torch.cat([b[:, :7] for b in boxes]).to(dev, torch.float32).contiguous()
    gl = torch.cat([lab.reshape(-1) for lab in gt_labels]).to(dev, torch.int64).contiguous()
    return gt, gl, _offsets([b.shape[0] for b in boxes])


def centerpoint_targets(boxes, labels, sample_sizes, task_num_classes, pc_min, voxel_size, out_size_factor, feature_map_size,
                        gaussian_overlap, min_radius, max_objs, norm_bbox=True):
    """CenterHead.get_targets for the whole batch: boxes [N, 7|9] fp32 gravity-centred, labels int64 [N], the samples' boxes
    concatenated (sample_sizes: host ints, one per sample); task_num_classes: classes per task (task t owns the labels after those of the
    tasks before it); feature_map_size = (W, H) = grid_size[:2] // out_size_factor.  Returns four lists over tasks, the reference's
    shapes and dtypes: heatmap [B, ncls, H, W] f32, anno_box [B, max_objs, 10] f32, ind [B, max_objs] int64, mask [B, max_objs] uint8.
    No host sync; bit-identical from run to run."""
    if not isinstance(boxes, torch.Tensor) or not boxes.is_cuda or not isinstance(labels, torch.Tensor) or not labels.is_cuda:
        raise L.SSTB200Error("centerpoint_targets: boxes and labels must be CUDA tensors (there is no CPU path)")
    if boxes.dtype != torch.float32:
        raise L.SSTB200Error(f"centerpoint_targets: boxes must be float32, got {boxes.dtype}")
    if boxes.dim() != 2 or boxes.shape[1] not in (7, 9):
        raise L.SSTB200Error(f"centerpoint_targets: boxes must be [N, 7] or [N, 9], got {tuple(boxes.shape)}")
    if labels.dim() != 1 or labels.shape[0] != boxes.shape[0]:
        raise L.SSTB200Error(f"centerpoint_targets: labels {tuple(labels.shape)} do not match boxes {tuple(boxes.shape)}")
    offsets = _sample_offsets("centerpoint_targets", sample_sizes, boxes.shape[0])
    W, H = (int(v) for v in feature_map_size)
    B, dev = len(offsets) - 1, boxes.device
    boxes, labels = boxes.contiguous(), labels.long().contiguous()
    task_off = _offsets(task_num_classes)
    hm = [torch.empty((B, int(n), H, W), dtype=torch.float32, device=dev) for n in task_num_classes]
    ab = [torch.empty((B, max_objs, 10), dtype=torch.float32, device=dev) for _ in task_num_classes]
    ind = [torch.empty((B, max_objs), dtype=torch.int64, device=dev) for _ in task_num_classes]
    mask = [torch.empty((B, max_objs), dtype=torch.uint8, device=dev) for _ in task_num_classes]
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_centerpoint_targets(
        c, L.ptr(boxes) if boxes.numel() else None, L.ptr(labels) if labels.numel() else None, boxes.shape[1],
        L.arr(C.c_int32, offsets), B, L.arr(C.c_int32, task_off), len(task_off) - 1, L.arr(C.c_float, [float(v) for v in pc_min[:2]]),
        L.arr(C.c_float, [float(v) for v in voxel_size[:2]]), int(out_size_factor), W, H, float(gaussian_overlap), int(min_radius),
        int(max_objs), int(bool(norm_bbox)), _ptrs(hm), _ptrs(ab), _ptrs(ind), _ptrs(mask)))
    return hm, ab, ind, mask


class GaussianFocalLossFunction(Function):
    """mmdet 2.14 GaussianFocalLoss (alpha 2, gamma 4, reduction 'mean', avg_factor = max(num_pos, 1)) on clip_sigmoid(logits): returns
    (loss, num_pos), both fp32 device scalars, num_pos = the number of target elements equal to 1.  Saves only the two inputs; the
    backward recomputes the per-element derivative.  As torch.clamp, the clamp keeps NaN: a NaN logit makes the loss NaN and its own
    gradient NaN."""

    @staticmethod
    def forward(ctx, logits, target, loss_weight=1.0):
        x, t = _fp32_cuda("logits", logits), _fp32_cuda("target", target)
        if x.shape != t.shape or x.numel() == 0:
            raise L.SSTB200Error(f"gaussian_focal_loss: logits {tuple(x.shape)} and target {tuple(t.shape)} must be one non-empty shape")
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        num_pos = torch.empty((), dtype=torch.float32, device=x.device)
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_gaussian_focal_loss_forward(c, L.ptr(x), L.ptr(t), x.numel(), float(loss_weight), L.ptr(loss),
                                                               L.ptr(num_pos)))
        ctx.save_for_backward(x, t, num_pos)
        ctx.loss_weight, ctx.in_dtype = float(loss_weight), logits.dtype
        ctx.mark_non_differentiable(num_pos)
        return loss, num_pos

    @staticmethod
    def backward(ctx, grad_loss, _grad_num_pos=None):
        x, t, num_pos = ctx.saved_tensors
        g = torch.empty_like(x)
        gl = grad_loss.float().contiguous()
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_gaussian_focal_loss_backward(c, L.ptr(x), L.ptr(t), x.numel(), ctx.loss_weight, L.ptr(num_pos), L.ptr(gl),
                                                                L.ptr(g)))
        return g.to(ctx.in_dtype), None, None


def gaussian_focal_loss(logits, target, loss_weight=1.0):
    """(loss, num_pos) of GaussianFocalLossFunction"""
    return GaussianFocalLossFunction.apply(logits, target, loss_weight)


def _l1_geom(heads, anno_box, ind, mask):
    if len(heads) != 5:
        raise L.SSTB200Error("centerpoint_l1_loss: five heads (reg, height, dim, rot, vel) are needed")
    hs = [_fp32_cuda(name, h, 4) for (name, _), h in zip(CENTERPOINT_HEADS, heads)]
    B, _, H, W = hs[0].shape
    for (name, ch), h in zip(CENTERPOINT_HEADS, hs):
        if tuple(h.shape) != (B, ch, H, W):
            raise L.SSTB200Error(f"centerpoint_l1_loss: {name} must be {(B, ch, H, W)}, got {tuple(h.shape)}")
    ab = _fp32_cuda("anno_box", anno_box, 3)
    M = ab.shape[1]
    if tuple(ab.shape) != (B, M, 10) or tuple(ind.shape) != (B, M) or tuple(mask.shape) != (B, M):
        raise L.SSTB200Error(f"centerpoint_l1_loss: anno_box {tuple(ab.shape)}, ind {tuple(ind.shape)} and mask {tuple(mask.shape)} do "
                             f"not fit [{B}, max_objs, 10] / [{B}, max_objs]")
    if not ind.is_cuda or not mask.is_cuda or ind.dtype != torch.int64 or mask.dtype not in (torch.uint8, torch.bool):
        raise L.SSTB200Error("centerpoint_l1_loss: ind must be int64 and mask uint8, on the GPU")
    return hs, ab, ind.contiguous(), mask.contiguous().view(torch.uint8), (B, H, W, M)


class CenterPointL1LossFunction(Function):
    """CenterHead.loss's regression term: mmdet 2.14 L1Loss (reduction 'mean') of anno_box [B, M, 10] against the five heads gathered
    at ind, weight mask * (target not NaN) * code_weights, avg_factor = sum(mask) + 1e-4 on the device.  The heads are read in place;
    the backward writes their dense gradients with each cell's objects summed in slot order (deterministic, no float atomics).  As in
    the reference, every slot is gathered, masked or not: a NaN target, or a NaN prediction at any slot's ind, makes the loss NaN, while
    the gradient there stays 0 (torch.sign(NaN) = 0)."""

    @staticmethod
    def forward(ctx, anno_box, ind, mask, code_weights, loss_weight, *heads):
        hs, ab, ind, mask, (B, H, W, M) = _l1_geom(heads, anno_box, ind, mask)
        cw = L.arr(C.c_float, [float(v) for v in code_weights])
        if len(cw) != 10:
            raise L.SSTB200Error(f"centerpoint_l1_loss: 10 code weights are needed, got {len(cw)}")
        loss = torch.empty((), dtype=torch.float32, device=ab.device)
        c = L.ctx(ab.device)
        L.check(c, L.lib().sstb200_centerpoint_l1_loss_forward(c, _ptrs(hs), B, H, W, L.ptr(ab), L.ptr(ind), L.ptr(mask), M, cw,
                                                               float(loss_weight), L.ptr(loss)))
        ctx.save_for_backward(ab, ind, mask, *hs)
        ctx.cfg = (list(code_weights), float(loss_weight), [h.dtype for h in heads])
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        ab, ind, mask, *hs = ctx.saved_tensors
        code_weights, loss_weight, dtypes = ctx.cfg
        B, _, H, W = hs[0].shape
        grads = [torch.empty_like(h) for h in hs]
        gl = grad_loss.float().contiguous()
        c = L.ctx(ab.device)
        L.check(c, L.lib().sstb200_centerpoint_l1_loss_backward(c, _ptrs(hs), B, H, W, L.ptr(ab), L.ptr(ind), L.ptr(mask), ab.shape[1],
                                                                L.arr(C.c_float, code_weights), loss_weight, L.ptr(gl), _ptrs(grads)))
        return (None, None, None, None, None) + tuple(g.to(d) for g, d in zip(grads, dtypes))


def centerpoint_l1_loss(preds, anno_box, ind, mask, code_weights, loss_weight=1.0):
    """preds: a dict with 'reg', 'height', 'dim', 'rot', 'vel' [B, C, H, W] -> the loss (fp32 device scalar)"""
    return CenterPointL1LossFunction.apply(anno_box, ind, mask, code_weights, loss_weight, *[preds[k] for k, _ in CENTERPOINT_HEADS])


# ----------------------------------------------------------------------------------------------
# Anchor3DHead training (mmdet3d/models/dense_heads/anchor3d_head.py:197-379, train_mixins.py:11-346)
# ----------------------------------------------------------------------------------------------
L.SIGNATURES["sstb200_anchor3d_targets"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.c_int, L.vp, L.vp, C.c_int, L.vp, C.c_int, L.vp, L.vp,
                                                      L.P_i32, C.c_int, L.P_f32, L.P_f32, L.P_f32, L.P_i32, C.c_int, C.c_int, C.c_float,
                                                      L.vp, L.vp, L.vp, L.vp, L.vp, L.vp, L.vp])
_FOCAL_ARGS = [L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, L.vp, L.vp, L.vp, C.c_float]
L.SIGNATURES["sstb200_anchor_focal_loss_forward"] = (C.c_int, _FOCAL_ARGS + [L.vp])
L.SIGNATURES["sstb200_anchor_focal_loss_backward"] = (C.c_int, _FOCAL_ARGS + [L.vp, L.vp])
_REG_ARGS = [L.vp, L.vp, L.vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, L.vp, L.vp, L.vp, L.vp, L.vp, L.P_f32, L.vp, C.c_float,
             C.c_float]
L.SIGNATURES["sstb200_anchor_reg_dir_loss_forward"] = (C.c_int, _REG_ARGS + [L.vp, L.vp])
L.SIGNATURES["sstb200_anchor_reg_dir_loss_backward"] = (C.c_int, _REG_ARGS + [L.vp, L.vp, L.vp])


def anchor3d_targets(x_centers, y_centers, size_z, size_wlh, rotations, gt_boxes, gt_labels, sample_sizes, num_classes, pos_iou_thr,
                     neg_iou_thr, min_pos_iou, gt_max_assign_all=True, assign_per_class=False, dir_offset=0.0):
    """anchor_target_3d of one level (AlignedAnchor3DRangeGenerator anchors, one MaxIoUAssigner per size, PseudoSampler,
    DeltaXYZWLHRBBoxCoder) for the whole batch.  The anchors are given by their separable axes, all fp32 CUDA tensors: x_centers [W],
    y_centers [H], size_z [S], size_wlh [S, 3], rotations [R]; anchor ((y W + x) S + s) R + r.  gt_boxes [N, 7] fp32 bottom-centre and
    gt_labels [N] on the GPU, the samples concatenated (sample_sizes: host ints).  pos_iou_thr / neg_iou_thr / min_pos_iou /
    gt_max_assign_all: one value per size (or one for all).  Returns (labels int64 [B, A], label_weights [B, A], bbox_targets [B, A, 7],
    bbox_weights [B, A, 7], dir_targets int64 [B, A], dir_weights [B, A], num_total_pos int64 device scalar), the reference's tensors in
    its anchor order.  No host sync; bit-identical from run to run."""
    axes = [_fp32_cuda(n, t) for n, t in (("x_centers", x_centers), ("y_centers", y_centers), ("size_z", size_z),
                                          ("size_wlh", size_wlh), ("rotations", rotations))]
    xc, yc, sz, wlh, rot = axes
    W, H, S, R = xc.numel(), yc.numel(), sz.numel(), rot.numel()
    if wlh.numel() != 3 * S:
        raise L.SSTB200Error(f"anchor3d_targets: size_wlh must be [{S}, 3], got {tuple(wlh.shape)}")
    if not isinstance(gt_boxes, torch.Tensor) or not gt_boxes.is_cuda or not isinstance(gt_labels, torch.Tensor) or not gt_labels.is_cuda:
        raise L.SSTB200Error("anchor3d_targets: gt_boxes and gt_labels must be CUDA tensors (there is no CPU path)")
    if gt_boxes.dtype != torch.float32 or gt_boxes.dim() != 2 or gt_boxes.shape[1] != 7:
        raise L.SSTB200Error(f"anchor3d_targets: gt_boxes must be float32 [N, 7], got {gt_boxes.dtype} {tuple(gt_boxes.shape)}")
    if gt_labels.dim() != 1 or gt_labels.shape[0] != gt_boxes.shape[0]:
        raise L.SSTB200Error(f"anchor3d_targets: gt_labels {tuple(gt_labels.shape)} do not match gt_boxes {tuple(gt_boxes.shape)}")
    offsets = _sample_offsets("anchor3d_targets", sample_sizes, gt_boxes.shape[0])

    def per_size(name, v, ctype):
        vals = list(v) if isinstance(v, (list, tuple)) else [v] * S
        if len(vals) != S:
            raise L.SSTB200Error(f"anchor3d_targets: {name} needs {S} values, got {len(vals)}")
        return L.arr(ctype, [ctype(x).value if ctype is C.c_float else int(bool(x)) for x in vals])

    B, A, dev = len(offsets) - 1, H * W * S * R, xc.device
    gt, gl = gt_boxes.contiguous(), gt_labels.long().contiguous()
    labels = torch.empty((B, A), dtype=torch.int64, device=dev)
    label_weights = torch.empty((B, A), dtype=torch.float32, device=dev)
    bbox_targets = torch.empty((B, A, 7), dtype=torch.float32, device=dev)
    bbox_weights = torch.empty((B, A, 7), dtype=torch.float32, device=dev)
    dir_targets = torch.empty((B, A), dtype=torch.int64, device=dev)
    dir_weights = torch.empty((B, A), dtype=torch.float32, device=dev)
    num_total_pos = torch.empty((), dtype=torch.int64, device=dev)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_anchor3d_targets(
        c, L.ptr(xc), W, L.ptr(yc), H, L.ptr(sz), L.ptr(wlh), S, L.ptr(rot), R, L.ptr(gt) if gt.numel() else None,
        L.ptr(gl) if gl.numel() else None, L.arr(C.c_int32, offsets), B, per_size("pos_iou_thr", pos_iou_thr, C.c_float),
        per_size("neg_iou_thr", neg_iou_thr, C.c_float), per_size("min_pos_iou", min_pos_iou, C.c_float),
        per_size("gt_max_assign_all", gt_max_assign_all, C.c_int32), int(bool(assign_per_class)), int(num_classes), float(dir_offset),
        L.ptr(labels), L.ptr(label_weights), L.ptr(bbox_targets), L.ptr(bbox_weights), L.ptr(dir_targets), L.ptr(dir_weights),
        L.ptr(num_total_pos)))
    return labels, label_weights, bbox_targets, bbox_weights, dir_targets, dir_weights, num_total_pos


def _anchor_geom(name, t, num_anchors, per_anchor, B=None, H=None, W=None):
    t = _fp32_cuda(name, t, 4)
    b, ch, h, w = t.shape
    if ch != num_anchors * per_anchor or (B is not None and (b, h, w) != (B, H, W)):
        raise L.SSTB200Error(f"{name} must be [B, {num_anchors} x {per_anchor}, H, W] on one map, got {tuple(t.shape)}")
    return t


def _anchor_targets_check(name, B, A, labels, *ts):
    if tuple(labels.shape) != (B, A) or labels.dtype != torch.int64 or not labels.is_cuda:
        raise L.SSTB200Error(f"{name}: labels must be int64 [{B}, {A}] on the GPU, got {labels.dtype} {tuple(labels.shape)}")
    for t in ts:
        if not t.is_cuda or t.shape[:2] != (B, A):
            raise L.SSTB200Error(f"{name}: targets must be [{B}, {A}, ...] on the GPU, got {tuple(t.shape)}")


class AnchorFocalLossFunction(Function):
    """Anchor3DHead.loss_single's classification term: mmdet 2.14 FocalLoss(use_sigmoid=True, gamma 2, alpha 0.25) of cls_score
    [B, A_loc C, H, W], read in place (no permuted copy), against labels [B, A] (background = num_classes) weighted by label_weights,
    divided by the device num_total_pos and multiplied by loss_weight.  The log-sigmoid is the stable softplus form (mmdet's
    py_sigmoid_focal_loss), exact out to any logit; mmcv's CUDA kernel instead saturates near 87 beyond about +-17.  A NaN logit makes the
    loss NaN and its own gradient NaN."""

    @staticmethod
    def forward(ctx, cls_score, labels, label_weights, num_total_pos, num_classes, loss_weight=1.0):
        x = _fp32_cuda("cls_score", cls_score, 4)
        B, ch, H, W = x.shape
        if ch % num_classes:
            raise L.SSTB200Error(f"anchor_focal_loss: {ch} channels are not a multiple of {num_classes} classes")
        A_loc = ch // num_classes
        lw = _fp32_cuda("label_weights", label_weights)
        _anchor_targets_check("anchor_focal_loss", B, H * W * A_loc, labels, lw)
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_anchor_focal_loss_forward(c, L.ptr(x), B, A_loc, int(num_classes), H, W, L.ptr(labels), L.ptr(lw),
                                                             L.ptr(num_total_pos), float(loss_weight), L.ptr(loss)))
        ctx.save_for_backward(x, labels, lw, num_total_pos)
        ctx.cfg = (int(num_classes), float(loss_weight), cls_score.dtype)
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        x, labels, lw, ntp = ctx.saved_tensors
        num_classes, loss_weight, dtype = ctx.cfg
        B, ch, H, W = x.shape
        g = torch.empty_like(x)
        gl = grad_loss.float().contiguous()
        c = L.ctx(x.device)
        L.check(c, L.lib().sstb200_anchor_focal_loss_backward(c, L.ptr(x), B, ch // num_classes, num_classes, H, W, L.ptr(labels), L.ptr(lw),
                                                              L.ptr(ntp), loss_weight, L.ptr(gl), L.ptr(g)))
        return g.to(dtype), None, None, None, None, None


def anchor_focal_loss(cls_score, labels, label_weights, num_total_pos, num_classes, loss_weight=1.0):
    """the loss (fp32 device scalar) of AnchorFocalLossFunction"""
    return AnchorFocalLossFunction.apply(cls_score, labels, label_weights, num_total_pos, num_classes, loss_weight)


class AnchorRegDirLossFunction(Function):
    """Anchor3DHead.loss_single's box and direction terms over the positives (0 <= label < num_classes): mmdet 2.14 L1Loss of bbox_pred
    [B, A_loc 7, H, W] against bbox_targets, weighted by bbox_weights * code_weight, with add_sin_difference on the yaw; and
    CrossEntropyLoss(use_sigmoid=False) of dir_cls_preds [B, A_loc 2, H, W] against dir_targets weighted by dir_weights.  Both divided by
    the device num_total_pos and multiplied by their loss weights; both heads are read in place.  Returns (loss_bbox, loss_dir); with no
    positive both are 0 with zero gradients, as the reference's pos_bbox_pred.sum().  The backward writes both gradients in full with no
    atomics: every positive anchor owns its own channels."""

    @staticmethod
    def forward(ctx, bbox_pred, dir_cls_preds, labels, bbox_targets, bbox_weights, dir_targets, dir_weights, num_total_pos, num_classes,
                code_weight, loss_weight_bbox, loss_weight_dir):
        p = _fp32_cuda("bbox_pred", bbox_pred, 4)
        B, ch, H, W = p.shape
        if ch % 7:
            raise L.SSTB200Error(f"anchor_reg_dir_loss: bbox_pred has {ch} channels, not a multiple of 7")
        A_loc = ch // 7
        d = _anchor_geom("dir_cls_preds", dir_cls_preds, A_loc, 2, B, H, W)
        bt, bw, dw = (_fp32_cuda(n, t) for n, t in (("bbox_targets", bbox_targets), ("bbox_weights", bbox_weights),
                                                     ("dir_weights", dir_weights)))
        _anchor_targets_check("anchor_reg_dir_loss", B, H * W * A_loc, labels, bt, bw, dir_targets, dw)
        if dir_targets.dtype != torch.int64 or bt.shape[-1] != 7 or bw.shape[-1] != 7:
            raise L.SSTB200Error("anchor_reg_dir_loss: dir_targets must be int64 and the box targets / weights [B, A, 7]")
        cw = [float(v) for v in (code_weight if code_weight else [1.0] * 7)]
        if len(cw) != 7:
            raise L.SSTB200Error(f"anchor_reg_dir_loss: 7 code weights are needed, got {len(cw)}")
        lb = torch.empty((), dtype=torch.float32, device=p.device)
        ld = torch.empty((), dtype=torch.float32, device=p.device)
        dt = dir_targets.contiguous()
        c = L.ctx(p.device)
        L.check(c, L.lib().sstb200_anchor_reg_dir_loss_forward(c, L.ptr(p), L.ptr(d), B, A_loc, int(num_classes), H, W, L.ptr(labels),
                                                               L.ptr(bt), L.ptr(bw), L.ptr(dt), L.ptr(dw), L.arr(C.c_float, cw),
                                                               L.ptr(num_total_pos), float(loss_weight_bbox), float(loss_weight_dir),
                                                               L.ptr(lb), L.ptr(ld)))
        ctx.save_for_backward(p, d, labels, bt, bw, dt, dw, num_total_pos)
        ctx.cfg = (int(num_classes), cw, float(loss_weight_bbox), float(loss_weight_dir), bbox_pred.dtype, dir_cls_preds.dtype)
        return lb, ld

    @staticmethod
    def backward(ctx, grad_bbox, grad_dir):
        p, d, labels, bt, bw, dt, dw, ntp = ctx.saved_tensors
        num_classes, cw, wb, wd, pdt, ddt = ctx.cfg
        B, ch, H, W = p.shape
        zero = torch.zeros((), dtype=torch.float32, device=p.device)
        gl = torch.stack([zero if grad_bbox is None else grad_bbox.float(), zero if grad_dir is None else grad_dir.float()]).contiguous()
        gp, gd = torch.empty_like(p), torch.empty_like(d)
        c = L.ctx(p.device)
        L.check(c, L.lib().sstb200_anchor_reg_dir_loss_backward(c, L.ptr(p), L.ptr(d), B, ch // 7, num_classes, H, W, L.ptr(labels),
                                                                L.ptr(bt), L.ptr(bw), L.ptr(dt), L.ptr(dw), L.arr(C.c_float, cw),
                                                                L.ptr(ntp), wb, wd, L.ptr(gl), L.ptr(gp), L.ptr(gd)))
        return (gp.to(pdt), gd.to(ddt)) + (None,) * 10


def anchor_reg_dir_loss(bbox_pred, dir_cls_preds, labels, bbox_targets, bbox_weights, dir_targets, dir_weights, num_total_pos, num_classes,
                        code_weight=None, loss_weight_bbox=1.0, loss_weight_dir=1.0):
    """(loss_bbox, loss_dir), fp32 device scalars, of AnchorRegDirLossFunction"""
    return AnchorRegDirLossFunction.apply(bbox_pred, dir_cls_preds, labels, bbox_targets, bbox_weights, dir_targets, dir_weights,
                                          num_total_pos, num_classes, code_weight, loss_weight_bbox, loss_weight_dir)


# ----------------------------------------------------------------------------------------------
# VoteSegHead training (mmdet3d/models/decode_heads/segmentation_head.py:107-283)
# ----------------------------------------------------------------------------------------------
class _VoteSegCfg(C.Structure):
    _fields_ = [("num_classes", C.c_int32), ("use_softmax", C.c_int32), ("gamma", C.c_float), ("alpha", C.c_float),
                ("logit_scale", C.c_float), ("loss_weight", C.c_float), ("loss_weight_vote", C.c_float), ("class_weight", L.P_f32),
                ("num_groups", C.c_int32), ("group_masks", C.POINTER(C.c_uint64)), ("group_thresh", L.P_f32),
                ("num_entries", C.c_int32), ("entry_group", L.P_i32), ("entry_class", L.P_i32)]


_VS_ARGS = [L.vp, C.POINTER(_VoteSegCfg), L.vp, C.c_int64, L.vp, C.c_int64, C.c_int64, L.vp, L.vp, L.vp]
L.SIGNATURES["sstb200_voteseg_targets"] = (C.c_int, [L.vp, L.vp, C.c_int64, L.P_i32, L.vp, L.vp, L.P_i32, C.c_int, C.c_int, L.vp, L.vp,
                                                     L.vp])
L.SIGNATURES["sstb200_voteseg_loss_forward"] = (C.c_int, _VS_ARGS + [L.vp, L.vp, L.vp])
L.SIGNATURES["sstb200_voteseg_loss_backward"] = (C.c_int, _VS_ARGS + [L.vp, L.vp, L.vp, L.vp])


def voteseg_targets(points_list_or_cat, offsets, gt_boxes, gt_labels, num_classes):
    """VoteSegHead.get_targets for the whole batch in one launch.  points_list_or_cat: a list of [n_b, >= 3] fp32 CUDA tensors (offsets
    None), or their concatenation [N, >= 3] with offsets = the B + 1 host sample offsets (ints or a CPU tensor; read in place, any row
    stride).  gt_boxes: a list over samples of [G_b, >= 7] bottom-centre boxes (tensors or objects with `.tensor`, columns 0-6 used),
    gt_labels: a list of int64 [G_b] (a negative label marks an invalid box).  num_classes: the head's class count, the background label.
    Returns (labels int64 [N], vote_targets f32 [N, 3], vote_mask bool [N]), the reference's tensors bit for bit.  No host sync."""
    if isinstance(points_list_or_cat, (list, tuple)):
        if offsets is not None:
            raise L.SSTB200Error("voteseg_targets: offsets are given by the list of points; pass None")
        pts_list = [_fp32_cuda("points", p, 2) for p in points_list_or_cat]
        offs = _offsets([p.shape[0] for p in pts_list])
        pts = torch.cat(pts_list) if len(pts_list) > 1 else pts_list[0]
    else:
        pts = points_list_or_cat
        if not isinstance(pts, torch.Tensor) or not pts.is_cuda or pts.dtype != torch.float32 or pts.dim() != 2:
            raise L.SSTB200Error("voteseg_targets: points must be a float32 [N, >= 3] CUDA tensor or a list of them")
        if isinstance(offsets, torch.Tensor):
            if offsets.is_cuda:
                raise L.SSTB200Error("voteseg_targets: offsets must be host values (reading device offsets would synchronise)")
            offsets = offsets.tolist()
        offs = [int(v) for v in offsets]
    if pts.shape[1] < 3 or pts.stride(1) != 1:
        if pts.shape[1] < 3:
            raise L.SSTB200Error(f"voteseg_targets: points need at least 3 columns, got {tuple(pts.shape)}")
        pts = pts.contiguous()
    B = len(offs) - 1
    if B < 1 or offs[0] != 0 or offs[-1] != pts.shape[0] or any(b < a for a, b in zip(offs, offs[1:])):
        raise L.SSTB200Error(f"voteseg_targets: offsets {offs} do not partition the {pts.shape[0]} points")
    if len(gt_boxes) != B or len(gt_labels) != B:
        raise L.SSTB200Error(f"voteseg_targets: {len(gt_boxes)} box and {len(gt_labels)} label lists for {B} samples")
    dev = pts.device
    gt, gl, gt_offs = _cat_gt("voteseg_targets", gt_boxes, gt_labels, dev)
    N = pts.shape[0]
    labels = torch.empty((N,), dtype=torch.int64, device=dev)
    vote_targets = torch.empty((N, 3), dtype=torch.float32, device=dev)
    vote_mask = torch.empty((N,), dtype=torch.bool, device=dev)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_voteseg_targets(c, L.ptr(pts) if N else None, pts.stride(0), L.arr(C.c_int32, offs),
                                               L.ptr(gt) if gt.numel() else None, L.ptr(gl) if gl.numel() else None,
                                               L.arr(C.c_int32, gt_offs), B, int(num_classes),
                                               L.ptr(labels) if N else None, L.ptr(vote_targets) if N else None,
                                               L.ptr(vote_mask) if N else None))
    return labels, vote_targets, vote_mask


class VoteSegLossConfig:
    """The constant part of VoteSegHead.losses: the loss settings and the training-log groups.  num_classes = logit columns C.
    Sigmoid heads: score_thresh[i] / class_names[i] give recall_<name> of class i.  Softmax heads: group_names (lists of class names) with
    one score_thresh each give the group scores of gather_group_by_names, recall_<name> of every grouped class and num_fg."""

    def __init__(self, num_classes, use_sigmoid, gamma=2.0, alpha=0.25, class_weight=None, logit_scale=1.0, loss_weight=1.0,
                 loss_weight_vote=1.0, score_thresh=None, class_names=None, group_names=None):
        self.num_classes, self.use_sigmoid = int(num_classes), bool(use_sigmoid)
        groups, entries, names = [], [], []   # (mask, thr); (group, class); recall key per entry
        if score_thresh is not None:
            if self.use_sigmoid:
                for i, thr in enumerate(score_thresh):
                    groups.append((1 << i, float(thr)))
                    entries.append((i, i))
                    names.append(class_names[i])
            else:
                for gi, g in enumerate(group_names):
                    idx = [list(class_names).index(n) for n in g]
                    mask = 0
                    for k in idx:
                        mask |= 1 << k
                    groups.append((mask, float(score_thresh[gi])))
                    for n, k in zip(g, idx):
                        entries.append((gi, k))
                        names.append(n)
        self.entry_names, self.log_fg = names, score_thresh is not None and not self.use_sigmoid
        cw = None if class_weight is None else [float(w) for w in class_weight]
        if cw is not None and len(cw) != self.num_classes:
            raise L.SSTB200Error(f"voteseg_loss: {len(cw)} class weights for {self.num_classes} classes")
        self.gamma, self.alpha, self.class_weight, self.logit_scale = float(gamma), float(alpha), cw, float(logit_scale)
        self.loss_weight, self.loss_weight_vote, self.groups, self.entries = float(loss_weight), float(loss_weight_vote), groups, entries

    def struct(self):
        """(sstb200_voteseg_cfg, the host arrays it points to: keep both alive over the call)"""
        keep = (L.arr(C.c_float, self.class_weight) if self.class_weight else None, L.arr(C.c_uint64, [m for m, _ in self.groups]),
                L.arr(C.c_float, [t for _, t in self.groups]), L.arr(C.c_int32, [g for g, _ in self.entries]),
                L.arr(C.c_int32, [k for _, k in self.entries]))
        s = _VoteSegCfg(self.num_classes, int(not self.use_sigmoid), self.gamma, self.alpha, self.logit_scale, self.loss_weight,
                        self.loss_weight_vote, keep[0], len(self.groups), keep[1], keep[2], len(self.entries), keep[3], keep[4])
        return s, keep

    def metrics(self, counts):
        """{recall_<name>: tp / (real + 1e-5)} and, for softmax heads, num_fg [1], as the reference's fp32 device tensors"""
        E = len(self.entry_names)
        out = {}
        if E == 0 and not self.log_fg:
            return out
        cf = counts.float()
        for e, name in enumerate(self.entry_names):
            out[f"recall_{name}"] = cf[e] / (cf[E + e] + 1e-5)
        if self.log_fg:
            out["num_fg"] = cf[2 * E:2 * E + 1]
        return out


def _row_major(name, t, cols):
    """t as fp32 [N, cols] rows with unit column stride, read in place when it already is"""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise L.SSTB200Error(f"{name} must be a CUDA tensor (there is no CPU path)")
    if t.dtype == torch.float16:                       # @force_fp32 casts half predictions
        t = t.float()
    if t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != cols:
        raise L.SSTB200Error(f"{name} must be float32 [N, {cols}], got {t.dtype} {tuple(t.shape)}")
    if t.stride(1) != 1 or t.stride(0) < cols:
        t = t.contiguous()
    return t


class VoteSegLossFunction(Function):
    """VoteSegHead.losses' two losses and training-log counts in one pass over the point rows (sstb200_voteseg_loss_forward): returns
    (losses [2] = (loss_sem_seg, loss_vote), counts int64 [2 E + 1], non-differentiable).  seg_logits [N, C] and vote_preds [N, 3 C] are
    read in place with their row strides; labels / vote_targets / vote_mask come from voteseg_targets.  Saves only the two predictions,
    the targets and the device n_valid; the backward writes each point's own rows with no atomics (bit-identical from run to run).  No
    host sync.  A NaN logit makes loss_sem_seg NaN and its own gradient NaN (its row's in softmax mode), not the whole gradient."""

    @staticmethod
    def forward(ctx, seg_logits, vote_preds, labels, vote_targets, vote_mask, cfg):
        Cn = cfg.num_classes
        x, v = _row_major("seg_logits", seg_logits, Cn), _row_major("vote_preds", vote_preds, 3 * Cn)
        N = x.shape[0]
        t = _fp32_cuda("vote_targets", vote_targets, 2)
        if v.shape[0] != N or t.shape != (N, 3) or labels.shape != (N,) or vote_mask.shape != (N,) or N == 0:
            raise L.SSTB200Error(f"voteseg_loss: logits {tuple(x.shape)}, vote_preds {tuple(v.shape)}, labels {tuple(labels.shape)}, "
                                 f"vote_targets {tuple(t.shape)} and vote_mask {tuple(vote_mask.shape)} do not fit N > 0 points")
        if labels.dtype != torch.int64 or not labels.is_cuda or vote_mask.dtype not in (torch.bool, torch.uint8) or not vote_mask.is_cuda:
            raise L.SSTB200Error("voteseg_loss: labels must be int64 and vote_mask bool, on the GPU")
        lab, m = labels.contiguous(), vote_mask.contiguous().view(torch.uint8)
        losses = torch.empty((2,), dtype=torch.float32, device=x.device)
        num_valid = torch.empty((), dtype=torch.int64, device=x.device)
        counts = torch.empty((2 * len(cfg.entry_names) + 1,), dtype=torch.int64, device=x.device)
        c = L.ctx(x.device)
        st, _keep = cfg.struct()
        L.check(c, L.lib().sstb200_voteseg_loss_forward(c, C.byref(st), L.ptr(x), x.stride(0), L.ptr(v), v.stride(0), N, L.ptr(lab),
                                                        L.ptr(t), L.ptr(m), L.ptr(losses), L.ptr(num_valid), L.ptr(counts)))
        ctx.save_for_backward(x, v, lab, t, m, num_valid)
        ctx.cfg, ctx.dtypes = cfg, (seg_logits.dtype, vote_preds.dtype)
        ctx.mark_non_differentiable(counts)
        return losses, counts

    @staticmethod
    def backward(ctx, grad_losses, _grad_counts=None):
        x, v, lab, t, m, num_valid = ctx.saved_tensors
        cfg = ctx.cfg
        N = x.shape[0]
        gx = torch.empty((N, cfg.num_classes), dtype=torch.float32, device=x.device)
        gv = torch.empty((N, 3 * cfg.num_classes), dtype=torch.float32, device=x.device)
        gl = grad_losses.float().contiguous()
        c = L.ctx(x.device)
        st, _keep = cfg.struct()
        L.check(c, L.lib().sstb200_voteseg_loss_backward(c, C.byref(st), L.ptr(x), x.stride(0), L.ptr(v), v.stride(0), N, L.ptr(lab),
                                                         L.ptr(t), L.ptr(m), L.ptr(num_valid), L.ptr(gl), L.ptr(gx), L.ptr(gv)))
        return gx.to(ctx.dtypes[0]), gv.to(ctx.dtypes[1]), None, None, None, None


def voteseg_loss(seg_logits, vote_preds, labels, vote_targets, vote_mask, cfg=None, **kwargs):
    """(loss_sem_seg, loss_vote, metrics) of VoteSegLossFunction: two fp32 device scalars carrying gradients and a dict of
    non-differentiable device tensors (recall_<name>, num_fg).  cfg: a VoteSegLossConfig, or its keyword arguments."""
    if cfg is None:
        cfg = VoteSegLossConfig(**kwargs)
    losses, counts = VoteSegLossFunction.apply(seg_logits, vote_preds, labels, vote_targets, vote_mask, cfg)
    return losses[0], losses[1], cfg.metrics(counts)


# ----------------------------------------------------------------------------------------------
# SparseClusterHeadV2 training (mmdet3d/models/dense_heads/sparse_cluster_head{,_v2}.py)
# ----------------------------------------------------------------------------------------------
class _ClusterHeadCfg(C.Structure):
    _fields_ = [("gamma", C.c_float), ("alpha", C.c_float), ("smooth_l1", C.c_int32), ("beta", C.c_float),
                ("loss_weight_cls", C.c_float), ("loss_weight_center", C.c_float), ("loss_weight_size", C.c_float),
                ("loss_weight_rot", C.c_float)]


_CH_ARGS = [L.vp, C.POINTER(_ClusterHeadCfg), C.c_int, C.c_int64, _PP, L.P_i64, L.P_i32, _PP, L.P_i64, _PP, _PP, L.vp, L.vp, L.vp]
L.SIGNATURES["sstb200_cluster_head_targets"] = (C.c_int, [L.vp, L.vp, C.c_int64, L.vp, C.c_int64, C.c_int64, L.vp, L.vp, L.P_i32, C.c_int,
                                                          C.c_int, L.P_i32, L.P_i32, C.c_int, L.P_i32, _PP, _PP, L.vp])
L.SIGNATURES["sstb200_cluster_head_loss_forward"] = (C.c_int, _CH_ARGS + [L.vp])
L.SIGNATURES["sstb200_cluster_head_loss_backward"] = (C.c_int, _CH_ARGS + [L.vp, _PP, _PP])

CLUSTER_HEAD_CODE_SIZE = 8


def _batch_index(cluster_inds, M):
    """the cluster batch index read in place: column 1 of int64 cluster_inds [M, 3], or a 1-D int64 index -> (tensor, element stride)"""
    if not isinstance(cluster_inds, torch.Tensor) or not cluster_inds.is_cuda or cluster_inds.dtype != torch.int64:
        raise L.SSTB200Error("cluster_head_targets: cluster_inds must be an int64 CUDA tensor")
    if cluster_inds.dim() == 2:
        if cluster_inds.shape[1] < 2 or cluster_inds.shape[0] != M:
            raise L.SSTB200Error(f"cluster_head_targets: cluster_inds {tuple(cluster_inds.shape)} for {M} clusters")
        col = cluster_inds[:, 1]
    elif cluster_inds.dim() == 1 and cluster_inds.shape[0] == M:
        col = cluster_inds
    else:
        raise L.SSTB200Error(f"cluster_head_targets: cluster_inds {tuple(cluster_inds.shape)} for {M} clusters")
    if M and col.stride(0) < 1:
        col = col.contiguous()
    return col, max(col.stride(0), 1)


def cluster_head_targets(cluster_xyz, cluster_inds, gt_boxes, gt_labels, tasks, class_names):
    """SparseClusterHeadV2.get_targets of every task for the whole batch in one launch.  cluster_xyz fp32 [M, >= 3] (read in place, any
    row stride); cluster_inds int64 [M, 3] (column 1 is the sample) or [M]; gt_boxes: a list over samples of [G_b, >= 7] bottom-centre
    boxes (tensors or objects with `.tensor`), gt_labels: a list of int64 [G_b] global class ids; tasks: lists of class names per task,
    class_names: the global class list.  Returns (labels, bbox_targets, num_pos): lists over tasks of int64 [M] (background = the task's
    class count), fp32 [M, 8] (zeros on negatives) and an int64 [T] device tensor of the positives.  A cluster whose sample index is
    outside [0, B) gets label -1 and NaN targets.  No host sync."""
    xyz = cluster_xyz
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] < 3:
        raise L.SSTB200Error("cluster_head_targets: cluster_xyz must be a float32 [M, >= 3] CUDA tensor")
    if xyz.stride(1) != 1 or xyz.stride(0) < 3:
        xyz = xyz.contiguous()
    M = xyz.shape[0]
    bidx, bstride = _batch_index(cluster_inds, M)
    if bidx.device != xyz.device:
        raise L.SSTB200Error(f"cluster_head_targets: cluster_inds on {bidx.device}, cluster_xyz on {xyz.device}")
    B = len(gt_boxes)
    if B < 1 or len(gt_labels) != B:
        raise L.SSTB200Error(f"cluster_head_targets: {len(gt_boxes)} box and {len(gt_labels)} label lists")
    names = list(class_names)
    class_task, class_rank = [-1] * len(names), [0] * len(names)
    for t, task in enumerate(tasks):
        for r, n in enumerate(task):
            k = names.index(n)
            class_task[k], class_rank[k] = t, r
    T = len(tasks)
    dev = xyz.device
    gt, gl, gt_offs = _cat_gt("cluster_head_targets", gt_boxes, gt_labels, dev)
    labels = [torch.empty((M,), dtype=torch.int64, device=dev) for _ in range(T)]
    targets = [torch.empty((M, CLUSTER_HEAD_CODE_SIZE), dtype=torch.float32, device=dev) for _ in range(T)]
    num_pos = torch.empty((T,), dtype=torch.int64, device=dev)
    c = L.ctx(dev)
    L.check(c, L.lib().sstb200_cluster_head_targets(
        c, L.ptr(xyz) if M else None, xyz.stride(0), L.ptr(bidx) if M else None, bstride, M, L.ptr(gt) if gt.numel() else None,
        L.ptr(gl) if gl.numel() else None, L.arr(C.c_int32, gt_offs), B, len(names),
        L.arr(C.c_int32, class_task), L.arr(C.c_int32, class_rank), T, L.arr(C.c_int32, [len(t) for t in tasks]), _ptrs(labels),
        _ptrs(targets), L.ptr(num_pos)))
    return labels, targets, num_pos


class ClusterHeadLossConfig:
    """The constant part of SparseClusterHeadV2.loss_single_task: the focal settings of loss_cls and the L1 / SmoothL1 settings and
    weights of loss_center / loss_size / loss_rot (the three must share their type and beta).  Built once per head."""

    def __init__(self, gamma=2.0, alpha=0.25, loss_weight_cls=1.0, loss_weight_center=1.0, loss_weight_size=1.0, loss_weight_rot=1.0,
                 smooth_l1=False, beta=1.0):
        self.gamma, self.alpha, self.smooth_l1, self.beta = float(gamma), float(alpha), bool(smooth_l1), float(beta)
        self.weights = (float(loss_weight_cls), float(loss_weight_center), float(loss_weight_size), float(loss_weight_rot))

    def struct(self):
        return _ClusterHeadCfg(self.gamma, self.alpha, int(self.smooth_l1), self.beta, *self.weights)


def _cluster_head_loss_inputs(labels, targets, num_pos, cls_avg, reg_avg, preds):
    """every tensor the loss kernels read as a raw device array, checked: the T cls_logits [M, C_t] and T reg_preds [M, 8] fp32 rows
    with unit column stride, labels int64 [M] and bbox_targets fp32 [M, 8] per task, num_pos int64 [T] and the fp32 avg factors [T],
    all CUDA tensors on the predictions' device.  Shapes and dtypes are checked before devices.  Returns them contiguous where the
    kernels need it."""
    T = len(labels)
    if T < 1 or len(targets) != T or len(preds) != 2 * T:
        raise L.SSTB200Error(f"cluster_head_loss: {len(preds)} predictions, {len(labels)} labels and {len(targets)} bbox_targets; "
                             "one cls_logits, reg_preds, labels and bbox_targets per task")
    for name, t in [("num_pos", num_pos), ("cls_avg_factor", cls_avg), ("reg_avg_factor", reg_avg)] + \
            [(f"labels[{k}]", a) for k, a in enumerate(labels)] + [(f"bbox_targets[{k}]", a) for k, a in enumerate(targets)] + \
            [(f"prediction {k}", a) for k, a in enumerate(preds)]:
        if not isinstance(t, torch.Tensor):
            raise L.SSTB200Error(f"cluster_head_loss: {name} must be a tensor, got {type(t).__name__}")
    M = preds[0].shape[0] if preds[0].dim() == 2 else -1
    if M < 1:
        raise L.SSTB200Error(f"cluster_head_loss: cls_logits[0] must be [M, C] with M > 0, got {tuple(preds[0].shape)}")
    for k in range(T):
        x, r = preds[k], preds[T + k]
        if x.dim() != 2 or x.shape[0] != M or x.shape[1] < 1 or r.shape != (M, CLUSTER_HEAD_CODE_SIZE):
            raise L.SSTB200Error(f"cluster_head_loss: task {k}: cls_logits {tuple(x.shape)} and reg_preds {tuple(r.shape)} do not fit "
                                 f"[{M}, C] and [{M}, {CLUSTER_HEAD_CODE_SIZE}]")
        if labels[k].dtype != torch.int64 or labels[k].shape != (M,):
            raise L.SSTB200Error(f"cluster_head_loss: labels[{k}] must be int64 [{M}], got {labels[k].dtype} {tuple(labels[k].shape)}")
        if targets[k].dtype != torch.float32 or targets[k].shape != (M, CLUSTER_HEAD_CODE_SIZE):
            raise L.SSTB200Error(f"cluster_head_loss: bbox_targets[{k}] must be float32 [{M}, {CLUSTER_HEAD_CODE_SIZE}], got "
                                 f"{targets[k].dtype} {tuple(targets[k].shape)}")
    if num_pos.dtype != torch.int64 or num_pos.shape != (T,):
        raise L.SSTB200Error(f"cluster_head_loss: num_pos must be int64 [{T}], got {num_pos.dtype} {tuple(num_pos.shape)}")
    for name, f in (("cls_avg_factor", cls_avg), ("reg_avg_factor", reg_avg)):
        if f.dtype not in (torch.float32, torch.float16) or f.shape != (T,):
            raise L.SSTB200Error(f"cluster_head_loss: {name} must be float32 [{T}], got {f.dtype} {tuple(f.shape)}")
    xs = [_row_major(f"cls_logits[{k}]", x, x.shape[1]) for k, x in enumerate(preds[:T])]
    rs = [_row_major(f"reg_preds[{k}]", r, CLUSTER_HEAD_CODE_SIZE) for k, r in enumerate(preds[T:])]
    dev = xs[0].device
    named = [(f"cls_logits[{k}]", a) for k, a in enumerate(xs)] + [(f"reg_preds[{k}]", a) for k, a in enumerate(rs)] + \
        [(f"labels[{k}]", a) for k, a in enumerate(labels)] + [(f"bbox_targets[{k}]", a) for k, a in enumerate(targets)] + \
        [("num_pos", num_pos), ("cls_avg_factor", cls_avg), ("reg_avg_factor", reg_avg)]
    for name, t in named:
        if not t.is_cuda or t.device != dev:
            raise L.SSTB200Error(f"cluster_head_loss: {name} is on {t.device}; every input must be a CUDA tensor on {dev}")
    labels = [a.contiguous() for a in labels]
    targets = [_fp32_cuda(f"bbox_targets[{k}]", a, 2) for k, a in enumerate(targets)]
    return (xs, rs, labels, targets, num_pos.contiguous(), _fp32_cuda("cls_avg_factor", cls_avg, 1),
            _fp32_cuda("reg_avg_factor", reg_avg, 1))


class ClusterHeadLossFunction(Function):
    """loss_single_task of every task in one launch sequence (sstb200_cluster_head_loss_forward): returns losses [T, 4] = (cls, center,
    size, rot) per task.  Inputs: cfg, the targets of cluster_head_targets, the device avg factors cls_avg [T] and reg_avg [T], then the
    T cls_logits [M, C_t] and the T reg_preds [M, 8], read in place with their row strides.  Saves the predictions, targets and factors
    only; the backward writes each cluster's own rows with no atomics (bit-identical from run to run).  No host sync."""

    @staticmethod
    def forward(ctx, cfg, labels, targets, num_pos, cls_avg, reg_avg, *preds):
        T = len(labels)
        xs, rs, labels, targets, num_pos, ca, ra = _cluster_head_loss_inputs(labels, targets, num_pos, cls_avg, reg_avg, preds)
        M = xs[0].shape[0]
        losses = torch.empty((T, 4), dtype=torch.float32, device=xs[0].device)
        c = L.ctx(xs[0].device)
        st = cfg.struct()
        args = (c, C.byref(st), T, M, _ptrs(xs), L.arr(C.c_int64, [x.stride(0) for x in xs]), L.arr(C.c_int32, [x.shape[1] for x in xs]),
                _ptrs(rs), L.arr(C.c_int64, [r.stride(0) for r in rs]), _ptrs(labels), _ptrs(targets), L.ptr(num_pos), L.ptr(ca), L.ptr(ra))
        L.check(c, L.lib().sstb200_cluster_head_loss_forward(*args, L.ptr(losses)))
        ctx.save_for_backward(num_pos, ca, ra, *xs, *rs, *labels, *targets)
        ctx.cfg, ctx.T, ctx.dtypes = cfg, T, [p.dtype for p in preds]
        return losses

    @staticmethod
    def backward(ctx, grad_losses):
        T = ctx.T
        saved = ctx.saved_tensors
        num_pos, ca, ra = saved[:3]
        xs, rs, labels, targets = saved[3:3 + T], saved[3 + T:3 + 2 * T], saved[3 + 2 * T:3 + 3 * T], saved[3 + 3 * T:]
        M = xs[0].shape[0]
        gx = [torch.empty((M, x.shape[1]), dtype=torch.float32, device=x.device) for x in xs]
        gr = [torch.empty((M, CLUSTER_HEAD_CODE_SIZE), dtype=torch.float32, device=x.device) for x in xs]
        gl = grad_losses.float().contiguous()
        c = L.ctx(xs[0].device)
        st = ctx.cfg.struct()
        L.check(c, L.lib().sstb200_cluster_head_loss_backward(
            c, C.byref(st), T, M, _ptrs(xs), L.arr(C.c_int64, [x.stride(0) for x in xs]), L.arr(C.c_int32, [x.shape[1] for x in xs]),
            _ptrs(rs), L.arr(C.c_int64, [r.stride(0) for r in rs]), _ptrs(labels), _ptrs(targets), L.ptr(num_pos), L.ptr(ca), L.ptr(ra),
            L.ptr(gl), _ptrs(gx), _ptrs(gr)))
        grads = [g.to(d) for g, d in zip(gx + gr, ctx.dtypes)]
        return (None, None, None, None, None, None, *grads)


def cluster_head_loss(cls_logits, reg_preds, labels, bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, cfg):
    """losses [T, 4] = (loss_cls, loss_center, loss_size, loss_rot) per task of ClusterHeadLossFunction, an fp32 device tensor carrying
    gradients to the T cls_logits and T reg_preds.  cls_avg_factor / reg_avg_factor: fp32 device [T] (see SparseClusterHeadV2.loss for
    how the head forms them).  A misshapen, mistyped or off-device input raises SSTB200Error."""
    if len(cls_logits) != len(labels) or len(reg_preds) != len(labels) or len(bbox_targets) != len(labels):
        raise L.SSTB200Error("cluster_head_loss: one cls_logits, reg_preds, labels and bbox_targets per task")
    return ClusterHeadLossFunction.apply(cfg, list(labels), list(bbox_targets), num_pos, cls_avg_factor, reg_avg_factor, *cls_logits,
                                         *reg_preds)
