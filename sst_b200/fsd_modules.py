"""FSD on libsstb200 (SURVEY 8f next-3): the instance grouping between the segmentation / voting head and the SIR backbone, and the RoI
point pooling of the second stage (DynamicPointROIExtractor, at the end of this file).  Mirrors mmdet3d/models/detectors/single_stage_fsd.py:28-81 (filter_almost_empty, find_connected_componets*),
:144-151 (modify_cluster_by_class) and :922-999 (ClusterAssigner) by name, arguments and return values.

The reference builds a dense n x n distance matrix per sample and labels it with scipy on the CPU (training and, by default, eval;
TorchEx `connected_components` when gpu_clustering is set).  Here: sstb200_connected_components - a cell grid from the bitmap-rank
index, a 3 x 3 neighbourhood test with the reference's fp32 distance arithmetic, lock-free union-find with smallest-index roots and a
bitmap rank for scipy's component numbering.  Labels are bit-identical to the reference's.  No CPU / PyTorch fallback."""
import ctypes as C

import torch
from torch import nn

from . import _lib as L
from . import ops
from .ops import scatter_v2, unique_rows
from .registry import ROI_EXTRACTORS

L.SIGNATURES["sstb200_connected_components"] = (C.c_int, [L.vp, L.vp, C.c_int, L.vp, C.c_int, C.c_int, C.c_float, L.P_f32, L.P_f32, L.vp, L.vp,
                                                         L.P_i32])


def connected_components(points, batch_idx, dist, batch_size=None, xy_bounds=None):
    """labels [n] int32 + number of components.  points [n, >= 2] fp32 CUDA (x, y first)."""
    if not points.is_cuda:
        raise L.SSTB200Error("sst_b200 connected_components needs CUDA tensors (no CPU fallback)")
    pts = points.float().contiguous()
    n = pts.shape[0]
    labels = torch.empty((n,), dtype=torch.int32, device=pts.device)
    if n == 0:
        return labels, 0
    bi = None if batch_idx is None else batch_idx.int().contiguous()
    if batch_size is None:
        batch_size = 1 if bi is None else int(bi.max().item()) + 1
    if xy_bounds is None:
        lo, hi = pts[:, :2].amin(0).tolist(), pts[:, :2].amax(0).tolist()
    else:
        lo, hi = xy_bounds
    num_dev = torch.empty((1,), dtype=torch.int32, device=pts.device)
    num_host = C.c_int32(0)
    c = L.ctx(pts.device)
    L.check(c, L.lib().sstb200_connected_components(c, pts.data_ptr(), pts.shape[1], L.ptr(bi), n, int(batch_size), float(dist),
                                                    L.arr(C.c_float, [float(v) for v in lo]), L.arr(C.c_float, [float(v) for v in hi]),
                                                    labels.data_ptr(), num_dev.data_ptr(), C.byref(num_host)))
    return labels, num_host.value


def filter_almost_empty(coors, min_points):
    """single_stage_fsd.py:28-32"""
    new_coors, unq_inv, unq_cnt = unique_rows(coors.long(), return_counts=True)
    return unq_cnt[unq_inv] >= min_points


def find_connected_componets(points, batch_idx, dist, xy_bounds=None):
    """single_stage_fsd.py:47-68 (per-sample scipy labelling with a running base) in one launch sequence"""
    assert len(points) > 0
    labels, _ = connected_components(points, batch_idx, dist, xy_bounds=xy_bounds)
    return labels


def find_connected_componets_single_batch(points, batch_idx, dist, xy_bounds=None):
    """single_stage_fsd.py:70-81: batch_idx is ignored (the reference's eval path assumes one sample)"""
    labels, _ = connected_components(points, None, dist, batch_size=1, xy_bounds=xy_bounds)
    return labels


find_connected_componets_gpu = find_connected_componets   # TorchEx cc_gpu(points, batch_idx, dist, 100, 2, False): same contract


def modify_cluster_by_class(cluster_inds_list):
    """single_stage_fsd.py:144-151: prepend the class id column"""
    return [torch.cat([inds.new_ones((len(inds), 1)) * i, inds], 1) for i, inds in enumerate(cluster_inds_list)]


class ClusterAssigner(nn.Module):
    """single_stage_fsd.py:922-999: per class, voxelise the voted centres (cluster_voxel_size), drop almost-empty voxels, average the
    centres per voxel (scatter_v2 'avg'), connect voxel centres closer than connected_dist in xy, and hand every point its
    (batch, cluster) pair."""

    def __init__(self, cluster_voxel_size, min_points, point_cloud_range, connected_dist, class_names=['Car', 'Cyclist', 'Pedestrian'],
                 gpu_clustering=(False, False)):
        super().__init__()
        self.cluster_voxel_size = cluster_voxel_size
        self.min_points = min_points
        self.connected_dist = connected_dist
        self.point_cloud_range = point_cloud_range
        self.class_names = class_names
        self.gpu_clustering = gpu_clustering
        self.num_classes = len(class_names)

    def _per_class(self, table, class_name):
        if isinstance(table, dict):
            return table[class_name]
        if isinstance(table, list):
            return table[self.class_names.index(class_name)]
        return table

    @torch.no_grad()
    def forward(self, points_list, batch_idx_list, gt_bboxes_3d=None, gt_labels_3d=None, origin_points=None):
        assert self.num_classes == len(self.class_names)
        origin_points = origin_points if origin_points is not None else [None] * len(points_list)
        res = [self.forward_single_class(p, b, n, o) for p, b, n, o in zip(points_list, batch_idx_list, self.class_names, origin_points)]
        cluster_inds_list, valid_mask_list = [r[0] for r in res], [r[1] for r in res]
        return modify_cluster_by_class(cluster_inds_list), valid_mask_list

    def forward_single_class(self, points, batch_idx, class_name, origin_points):
        batch_idx = batch_idx.int()
        voxel_size = torch.tensor(self._per_class(self.cluster_voxel_size, class_name), device=points.device)
        pc_range = torch.tensor(self.point_cloud_range, device=points.device)
        coors = torch.div(points - pc_range[None, :3], voxel_size[None, :], rounding_mode='floor').int()
        coors = torch.cat([batch_idx[:, None], coors], dim=1)
        valid_mask = filter_almost_empty(coors, min_points=self.min_points)
        if not valid_mask.any():
            valid_mask = ~valid_mask
        points, batch_idx, coors = points[valid_mask], batch_idx[valid_mask], coors[valid_mask]
        sampled_centers, voxel_coors, inv_inds = scatter_v2(points, coors, mode='avg', return_inv=True)
        dist = self._per_class(self.connected_dist, class_name)
        bounds = (self.point_cloud_range[0:2], self.point_cloud_range[3:5])
        if self.training or self.gpu_clustering[1]:
            cluster_inds = find_connected_componets(sampled_centers, voxel_coors[:, 0], dist, bounds)
        else:
            cluster_inds = find_connected_componets_single_batch(sampled_centers, voxel_coors[:, 0], dist, bounds)
        assert len(cluster_inds) == len(sampled_centers)
        cluster_inds_per_point = torch.stack([batch_idx, cluster_inds[inv_inds]], 1)
        return cluster_inds_per_point, valid_mask


@ROI_EXTRACTORS.register_module()
class DynamicPointROIExtractor(nn.Module):
    """dynamic_point_roi_extractor.py:9-136: the points of every RoI of FSD's second stage (roi_head of configs/fsd), through
    sstb200_dynamic_point_pool.  Returns (point index, RoI index, dict(local_xyz, boundary_offset, is_in_margin)).

    The reference loops over the samples, one op call each, adding running point / RoI bases.  Here the samples go through ONE call
    whose capacity (max_all_pts) and fake row (-1, -1, zeros for a sample without any pair) apply per sample, which gives the loop's
    output row for row.  As in the reference, every sample needs a RoI and a point, and the points are sorted by batch; the RoIs
    must be too (rois[:, 0] ascending), or the reference's bases would index the wrong rows."""

    def __init__(self, init_cfg=None, debug=True, extra_wlh=[0, 0, 0], max_inbox_point=512, max_all_pts=50000):
        super().__init__()
        self.init_cfg = init_cfg
        self.debug = debug
        self.extra_wlh = extra_wlh
        self.max_inbox_point = max_inbox_point
        self.max_all_pts = max_all_pts

    def forward(self, pts_xyz, batch_inds, rois, max_inbox_point=None, batch_size=None):
        if batch_size == 1:
            return self.fast_single_sample_forward(pts_xyz, rois, max_inbox_point)
        if not (pts_xyz.is_cuda and batch_inds.is_cuda and rois.is_cuda):
            raise L.SSTB200Error("sst_b200 DynamicPointROIExtractor needs CUDA tensors (no CPU fallback)")
        assert len(pts_xyz) > 0 and len(batch_inds) > 0 and len(rois) > 0
        if max_inbox_point is None:
            max_inbox_point = self.max_inbox_point
        pb, rb = batch_inds.int(), rois[:, 0].int()
        num = int(pb.max()) + 1
        stats = torch.cat([torch.stack([(pb[1:] >= pb[:-1]).all(), (rb[1:] >= rb[:-1]).all(), (rb >= 0).all(), (pb >= 0).all()]).int(),
                           torch.bincount(rb.clamp(0, num), minlength=num + 1)[:num].int(), torch.bincount(pb.clamp(0), minlength=num).int()])
        stats = stats.tolist()
        if not (stats[0] and stats[3]):
            raise ValueError("DynamicPointROIExtractor: batch_inds must be sorted and non-negative")
        if not (stats[1] and stats[2]):
            raise ValueError("DynamicPointROIExtractor: rois[:, 0] must be sorted (ascending, non-negative batch ids)")
        nroi, npts = stats[4:4 + num], stats[4 + num:]
        if min(nroi) == 0 or min(npts) == 0:
            raise ValueError(f"DynamicPointROIExtractor: every sample needs RoIs and points (RoIs {nroi}, points {npts})")
        used = sum(nroi)   # RoIs of batch ids past the points' are never visited by the reference loop
        all_inds, all_roi_inds, all_pts_info = ops.point_pool(rois[:used, 1:], rb[:used], pts_xyz, pb, self.extra_wlh, max_inbox_point,
                                                              self.max_all_pts, per_sample=True, num_samples=num)
        all_out_xyz = all_pts_info[:, :3]
        all_local_xyz = all_pts_info[:, 3:6]
        all_offset = all_pts_info[:, 6:-1]
        is_in_margin = all_pts_info[:, -1]
        if self.debug:   # dynamic_point_roi_extractor.py:92-101
            roi_per_pts = rois[..., 1:][all_roi_inds]
            in_box_pts = pts_xyz[all_inds]
            assert torch.isclose(in_box_pts, all_out_xyz).all()
            assert torch.isclose(all_offset[:, 0] + all_offset[:, 3], roi_per_pts[:, 4]).all()
            assert torch.isclose(all_offset[:, 1] + all_offset[:, 4], roi_per_pts[:, 3]).all()
            assert torch.isclose(all_offset[:, 2] + all_offset[:, 5], roi_per_pts[:, 5]).all()
            assert (all_local_xyz[:, 0].abs() < roi_per_pts[:, 4] + self.extra_wlh[0] + 1e-5).all()
            assert (all_local_xyz[:, 1].abs() < roi_per_pts[:, 3] + self.extra_wlh[1] + 1e-5).all()
            assert (all_local_xyz[:, 2].abs() < roi_per_pts[:, 5] + self.extra_wlh[2] + 1e-5).all()
        return all_inds, all_roi_inds, dict(local_xyz=all_local_xyz, boundary_offset=all_offset, is_in_margin=is_in_margin)

    def fast_single_sample_forward(self, pts_xyz, rois, max_inbox_point=None):
        """:111-136 (the op's default max_all_pts, as there)"""
        if max_inbox_point is None:
            max_inbox_point = self.max_inbox_point
        ext_pts_inds, roi_inds, ext_pts_info = ops.dynamic_point_pool(rois[..., 1:].contiguous(), pts_xyz.contiguous(), self.extra_wlh,
                                                                      max_inbox_point)
        return ext_pts_inds, roi_inds, dict(local_xyz=ext_pts_info[:, 3:6], boundary_offset=ext_pts_info[:, 6:-1],
                                            is_in_margin=ext_pts_info[:, -1])
