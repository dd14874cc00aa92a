"""FSDv2 virtual-voxel front (BASELINE config 5; SURVEY 8f): the data-parallel part of `SingleStageFSDV2.extract_feat`
(mmdet3d/models/detectors/single_stage_fsd_v2.py:157-271) - everything between the segmentor's outputs and the sparse-conv mixer, and
the mask / centre bookkeeping after it.  The detector class itself (heads, losses, grouping) is outside the hot path; this module
carries the same sub-module names (`virtual_proj`, `ori_proj`, `recover_proj`, `ms_projectors`, `voxel_encoder`) so that the
detector's state-dict entries for them load unchanged.

One voxel index serves the whole front: the `DynamicScatterVFE` call produces (voxel_coors, unq_inv) and the indicator / centroid
reductions reuse it (the reference calls torch.unique again inside every scatter_v2)."""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib as L
from . import ops
from .registry import build_backbone, build_voxel_encoder

L.SIGNATURES["sstb200_voxelize_with_batch_idx"] = (C.c_int, [L.vp, L.vp, C.c_int, C.c_int, L.vp, L.P_f32, L.P_f32, L.vp])


def voxelize_with_batch_idx(points, batch_idx, voxel_size, point_cloud_range):
    """single_stage_fsd_v2.py:108-123: [n,4] int64 (batch, z, y, x), torch.div(..., rounding_mode='floor') semantics, no clamp."""
    ops._need_cuda(points, batch_idx)
    assert points.dim() == 2 and points.shape[1] >= 3 and batch_idx.shape[0] == points.shape[0]
    pts = points.float()
    if pts.stride(1) != 1:
        pts = pts.contiguous()
    bi = batch_idx.long().contiguous()
    n = pts.shape[0]
    coors = torch.empty((n, 4), dtype=torch.int64, device=pts.device)
    c = L.ctx(pts.device)
    L.check(c, L.lib().sstb200_voxelize_with_batch_idx(c, pts.data_ptr(), n, pts.stride(0), bi.data_ptr(), L.arr(C.c_float, voxel_size),
                                                       L.arr(C.c_float, point_cloud_range[:3]), coors.data_ptr()))
    return coors


class VirtualVoxelFront(nn.Module):
    """Constructor kwargs = the corresponding kwargs of SingleStageFSDV2 (configs/fsdv2/*.py): `voxel_encoder` (a DynamicScatterVFE
    config), `virtual_point_projector`, `multiscale_cfg`, `point_cloud_range`, `train_cfg`.  In training mode `finish` also returns
    `virtual_centroid`, the mean of each virtual voxel's points (FSDV2Head's centroid_assign); train_cfg centroid_alpha, which no
    config sets, raises ValueError."""

    def __init__(self, voxel_encoder, virtual_point_projector, point_cloud_range=None, multiscale_cfg=None, as_rpn=False, backbone=None,
                 train_cfg=None):
        super().__init__()
        if train_cfg is not None and train_cfg.get("centroid_alpha", None) is not None:
            raise ValueError(f"VirtualVoxelFront: train_cfg centroid_alpha is not supported, got {train_cfg.get('centroid_alpha')}")
        self.voxel_encoder = build_voxel_encoder(voxel_encoder)
        self.backbone = build_backbone(backbone) if backbone is not None else None   # VirtualVoxelMixer (spconv_modules.py)
        self.virtual_voxel_size = voxel_encoder["voxel_size"]
        self.point_cloud_range = voxel_encoder["point_cloud_range"] if point_cloud_range is None else point_cloud_range
        vpp = virtual_point_projector
        self.virtual_proj = ops.build_mlp(vpp["in_channels"], vpp["hidden_dims"], vpp["norm_cfg"])
        self.ori_proj = ops.build_mlp(vpp["ori_in_channels"], vpp["ori_hidden_dims"], vpp["norm_cfg"])
        self.zero_virtual_feature = vpp.get("zero_virtual_feature", False)
        self.only_virtual = vpp.get("only_virtual", False)
        self.as_rpn = as_rpn
        if as_rpn:
            self.recover_proj = ops.build_mlp(vpp["recover_in_channels"], vpp["recover_hidden_dims"], vpp["norm_cfg"])
        self.multiscale_cfg = multiscale_cfg
        if multiscale_cfg is not None:
            self.ms_projectors = nn.ModuleList([ops.build_mlp(proj[0], proj[1:], multiscale_cfg["norm_cfg"])
                                                for proj in multiscale_cfg["projector_hiddens"]])

    # ---- single_stage_fsd_v2.py:108-131
    @torch.no_grad()
    def voxelize_with_batch_idx(self, points, batch_idx):
        return voxelize_with_batch_idx(points[:, :3], batch_idx, self.virtual_voxel_size, self.point_cloud_range)

    def clip_points(self, points, pc_range):
        eps = 1e-5
        lo = points.new_tensor([pc_range[0] + eps, pc_range[1] + eps, pc_range[2] + eps])
        hi = points.new_tensor([pc_range[3] - eps, pc_range[4] - eps, pc_range[5] - eps])
        points[:, :3] = torch.minimum(torch.maximum(points[:, :3], lo), hi)   # in place, like the reference
        return points

    # ---- single_stage_fsd_v2.py:398-434
    def ms_coors_proj(self, coors, sparse_shape):
        tgt = self.multiscale_cfg["target_sparse_shape"]
        bev_stride = tgt[1] // sparse_shape[1]
        assert bev_stride == tgt[2] / sparse_shape[2]
        z_stride = tgt[0] // sparse_shape[0]
        assert z_stride >= 1 and bev_stride >= 1
        mul = coors.new_tensor([1, z_stride, bev_stride, bev_stride])
        add = coors.new_tensor([0, z_stride // 2, bev_stride // 2, bev_stride // 2])
        return coors * mul + add

    # ---- single_stage_fsd_v2.py:375-396
    def multiscale_fusion(self, ms_data, voxel_feats, coors):
        """ms_data[l]: objects with `.features`, `.indices`, `.spatial_shape` (SparseConvTensor-like)."""
        cfg = self.multiscale_cfg
        ms_data = [ms_data[l] for l in cfg["multiscale_levels"]]
        ms_feats = [self.ms_projectors[i](ms_data[i].features) for i in range(len(ms_data))]
        ms_coors = [self.ms_coors_proj(d.indices.long(), d.spatial_shape) for d in ms_data]
        num_add = sum(len(f) for f in ms_feats)
        cat_feats = torch.cat([voxel_feats] + ms_feats, 0)
        cat_coors = torch.cat([coors] + ms_coors, 0)
        indicators = torch.cat([voxel_feats.new_ones(len(voxel_feats), 1), voxel_feats.new_zeros(num_add, 1)], 0)
        # one voxel index for both reductions
        out_feats, out_coors, inv = ops.scatter_v2(cat_feats, cat_coors, mode=cfg["fusion_mode"], return_inv=True)
        out_ind, _ = ops.scatter_v2(indicators, cat_coors, mode="max", return_inv=False, unq_inv=inv, new_coors=out_coors)
        singlescale_mask = out_ind.squeeze(1) == 1
        return out_feats, out_coors, singlescale_mask

    # ---- single_stage_fsd_v2.py:157-215: everything before `self.backbone(...)`
    def front(self, sampled_dict, origin_dict, multiscale_features=None):
        sampled_pts = sampled_dict["seg_points"]
        sampled_centers = self.clip_points(sampled_dict["center_preds"], self.point_cloud_range)
        offset = (sampled_centers - sampled_pts[:, :3]) / 10  # hardcoded normaliser of the reference
        proj_input = torch.cat([sampled_dict["seg_feats"], offset, sampled_dict["seg_logits"], sampled_pts[:, 3:]], 1)
        vir_pts_feat = self.virtual_proj(proj_input)
        if self.zero_virtual_feature:
            vir_pts_feat = vir_pts_feat * 0
        ori_pts = origin_dict["seg_points"]
        ori_pts_feat = self.ori_proj(origin_dict["seg_feats"])
        cat_pts = torch.cat([ori_pts[:, :3], sampled_centers], 0)
        cat_feat = torch.cat([ori_pts_feat, vir_pts_feat], 0)
        cat_batch_idx = torch.cat([origin_dict["batch_idx"], sampled_dict["batch_idx"]], 0)
        coors = self.voxelize_with_batch_idx(cat_pts, cat_batch_idx)
        voxel_feats, voxel_coors, unq_inv = self.voxel_encoder(torch.cat([cat_pts, cat_feat], 1), coors, return_inv=True)
        pts_indicators = torch.cat([cat_pts.new_zeros(len(ori_pts)), cat_pts.new_ones(len(sampled_centers))])
        voxel_indicators, _ = ops.scatter_v2(pts_indicators[:, None], coors, mode="avg", return_inv=False, unq_inv=unq_inv,
                                             new_coors=voxel_coors)
        virtual_mask = voxel_indicators.squeeze(1) > 0
        out = dict(voxel_feats=voxel_feats, voxel_coors=voxel_coors, unq_inv=unq_inv, virtual_mask=virtual_mask, coors=coors,
                   cat_pts=cat_pts, cat_batch_idx=cat_batch_idx, pts_indicators=pts_indicators, singlescale_mask=None,
                   encoder_coors=voxel_coors)   # the voxels unq_inv indexes, before multiscale fusion and only_virtual
        if multiscale_features is not None:
            out["voxel_feats"], out["voxel_coors"], out["singlescale_mask"] = self.multiscale_fusion(multiscale_features, voxel_feats,
                                                                                                      voxel_coors)
        if self.only_virtual:
            assert multiscale_features is None
            out["voxel_feats"] = out["voxel_feats"][virtual_mask]
            out["voxel_coors"] = out["voxel_coors"][virtual_mask]
        return out

    # ---- single_stage_fsd_v2.py:157-271: front -> sparse-conv mixer -> bookkeeping, eval mode
    def extract_feat(self, sampled_dict, origin_dict, gt_bboxes_3d=None, multiscale_features=None):
        assert self.backbone is not None, "built without a backbone: call front() / finish() around your own mixer"
        fr = self.front(sampled_dict, origin_dict, multiscale_features)
        batch_size = int(fr["coors"][:, 0].max().item()) + 1
        out_voxel_feats, out_coors, sparse_shape = self.backbone(fr["voxel_feats"], fr["voxel_coors"], batch_size)
        return self.finish(fr, out_voxel_feats, out_coors, sparse_shape)

    # ---- single_stage_fsd_v2.py:217-242, 262-269: after the backbone
    def finish(self, front_out, out_voxel_feats, out_coors, sparse_shape=None):
        virtual_mask = front_out["virtual_mask"]
        ssm = front_out["singlescale_mask"]
        if ssm is not None:
            out_voxel_feats, out_coors = out_voxel_feats[ssm], out_coors[ssm]
        vs = out_voxel_feats.new_tensor(self.virtual_voxel_size)
        lo = out_voxel_feats.new_tensor(self.point_cloud_range[:3])
        voxel_centers = (out_coors[:, [3, 2, 1]] + 0.5) * vs[None, :] + lo[None, :]
        if self.only_virtual:
            vf, vc, ce = out_voxel_feats, out_coors, voxel_centers
        else:
            vf, vc, ce = out_voxel_feats[virtual_mask], out_coors[virtual_mask], voxel_centers[virtual_mask]
        out = dict(virtual_feats=vf, virtual_coors=vc, virtual_centers=ce, sparse_shape=sparse_shape)
        if self.training:
            # single_stage_fsd_v2.py:246-261 without centroid_alpha: the mean of each voxel's points over the front's voxel index; the
            # reference's `.all()` assert that it lies in its voxel is dropped (a host sync)
            centroid, _ = ops.scatter_v2(front_out["cat_pts"][:, :3], front_out["coors"], mode="avg", return_inv=False,
                                         unq_inv=front_out["unq_inv"], new_coors=front_out["encoder_coors"])
            out["virtual_centroid"] = centroid[virtual_mask]
        if self.as_rpn:
            out["pts_feats"] = self.recover_point_features(out_voxel_feats, out_coors, front_out["cat_pts"], front_out["voxel_coors"]
                                                           if ssm is None else front_out["voxel_coors"][ssm], front_out["unq_inv"])
            out["pts_xyz"] = front_out["cat_pts"]
            out["pts_indicators"] = front_out["pts_indicators"]
            out["pts_batch_inds"] = front_out["cat_batch_idx"]
        return out

    # ---- single_stage_fsd_v2.py:133-155
    def recover_point_features(self, out_voxel_feats, out_coors, cat_pts, voxel_encoder_coors, voxel_encoder_inv):
        if out_coors.shape != voxel_encoder_coors.shape or not bool((out_coors == voxel_encoder_coors).all()):
            raise NotImplementedError("the mixer changed the voxel layout (the reference raises here as well)")
        vs = out_voxel_feats.new_tensor(self.virtual_voxel_size)
        lo = out_voxel_feats.new_tensor(self.point_cloud_range[:3])
        coors_per_pts = out_coors[voxel_encoder_inv]
        feat_per_pts = out_voxel_feats[voxel_encoder_inv]
        center_per_pts = (coors_per_pts[:, [3, 2, 1]] + 0.5) * vs[None, :] + lo[None, :]
        offset = (center_per_pts - cat_pts) / vs[None, :] * 2
        return self.recover_proj(torch.cat([feat_per_pts, offset], 1))
