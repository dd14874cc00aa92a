"""PartA2's RoI layer on libsstb200: Single3DRoIAwareExtractor (mmdet3d/models/roi_heads/roi_extractors/single_roiaware_extractor.py),
built on ops.RoIAwarePool3d.  The reference pools sample by sample, one op call each; here every sample goes through one
sstb200_roiaware_pool3d call with per-point and per-RoI batch ids, and the RoIs are ordered sample-major first, which gives the
reference's concatenation."""
import torch
from torch import nn

from . import _lib as L
from . import ops
from .registry import ROI_EXTRACTORS


@ROI_EXTRACTORS.register_module()
class Single3DRoIAwareExtractor(nn.Module):
    """single_roiaware_extractor.py:8-53.  roi_layer = dict(type='RoIAwarePool3d', out_size=..., max_pts_per_voxel=..., mode=...), built
    from the op namespace by `type` as there.  forward(feats [N, C], coordinate [N, 3], batch_inds [N], rois [K, 8] = (batch id, box))
    -> pooled [K', ox, oy, oz, C]: the RoIs of sample 0, then sample 1, ... up to max(batch_inds), each sample's RoIs in input order
    (RoIs of other batch ids are not pooled, as in the reference's loop)."""

    def __init__(self, roi_layer=None, init_cfg=None):
        super().__init__()
        self.init_cfg = init_cfg
        self.roi_layer = self.build_roi_layers(roi_layer)

    def build_roi_layers(self, layer_cfg):
        cfg = layer_cfg.copy()
        layer_type = cfg.pop('type')
        assert hasattr(ops, layer_type)
        return getattr(ops, layer_type)(**cfg)

    def forward(self, feats, coordinate, batch_inds, rois):
        if not (feats.is_cuda and coordinate.is_cuda and batch_inds.is_cuda and rois.is_cuda):
            raise L.SSTB200Error("sst_b200 Single3DRoIAwareExtractor needs CUDA tensors (no CPU fallback)")
        pb = batch_inds.int()
        rb = rois[..., 0].int()
        num = int(pb.max()) + 1
        keep = ((rb >= 0) & (rb < num)).nonzero()[:, 0]
        order = keep[torch.sort(rb[keep], stable=True).indices]       # sample-major, input order within a sample
        pb = torch.where(pb < 0, torch.full_like(pb, num), pb)         # a point of no listed sample pairs with no RoI
        layer = self.roi_layer
        return ops.RoIAwarePool3dFunction.apply(rois[order, 1:], coordinate, feats, layer.out_size, layer.max_pts_per_voxel, layer.mode,
                                                rb[order], pb)
