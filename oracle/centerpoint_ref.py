"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

The reference's own CenterHead (mmdet3d/models/dense_heads/centerpoint_head.py), imported unmodified for its training and decoding path
on the CPU: the real draw_heatmap_gaussian / gaussian_radius (core/utils/gaussian.py), clip_sigmoid (models/utils/clip_sigmoid.py),
xywhr2xyxyr (core/bbox/structures/utils.py) and CenterPointBBoxCoder (core/bbox/coders/centerpoint_bbox_coders.py); the mmdet 2.14
losses restated in oracle/centerpoint_oracle.py; nms_gpu from oracle/iou3d_oracle.py; mmcv's ConvModule and 'DCN' as
oracle/centerpoint_shim.py builds them.  The box stub gives `tensor` / `gravity_center` as LiDARInstance3DBoxes does."""
import importlib
import os
import sys
import types
from functools import partial

import torch
from torch import nn

from oracle import centerpoint_oracle as CO
from oracle import centerpoint_shim as CS
from oracle import iou3d_oracle as IO
from oracle.ref_shim import REF_ROOT, _Registry, available, load, reference_functions  # noqa: F401  (available: for the tests' skip)


class Boxes:
    """LiDARInstance3DBoxes as get_targets / get_bboxes use it: `tensor` (bottom-centre z), `gravity_center`, `bev`"""

    def __init__(self, tensor, box_dim=None):
        self.tensor = tensor

    @property
    def gravity_center(self):
        b = self.tensor
        return torch.cat([b[:, :2], b[:, 2:3] + b[:, 5:6] * 0.5], 1)

    @property
    def bev(self):
        return self.tensor[:, [0, 1, 3, 4, 6]]


class _GaussianFocalLoss(nn.Module):
    def __init__(self, reduction="mean", loss_weight=1.0, alpha=2.0, gamma=4.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        return self.loss_weight * CO.gaussian_focal_loss(pred, target).sum() / avg_factor


class _L1Loss(nn.Module):
    def __init__(self, reduction="mean", loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, pred, target, weight=None, avg_factor=None):
        return self.loss_weight * ((pred - target).abs() * weight).sum() / avg_factor


_LOSSES = {"GaussianFocalLoss": _GaussianFocalLoss, "L1Loss": _L1Loss}
_HEAD = None


def _multi_apply(func, *args, **kwargs):   # mmdet/core/utils/misc.py
    pfunc = partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def load_center_head():
    """namespace(CenterHead, CenterPointBBoxCoder, Boxes) of the reference, built on the CPU"""
    global _HEAD
    if _HEAD is not None:
        return _HEAD
    CS.load_centerpoint_head()       # the DCN / ConvModule stubs and the registry the separate heads are built from
    load()
    cnn = sys.modules["mmcv.cnn"]
    dense_build = cnn.build_conv_layer

    def build_conv_layer(cfg, *args, **kwargs):
        c = dict(cfg or dict(type="Conv2d"))
        if c.get("type") == "DCN":
            c.pop("type")
            return CS._OracleDCN(*args, **kwargs, **c)
        return dense_build(cfg, *args, **kwargs)

    gauss = reference_functions("mmdet3d/core/utils/gaussian.py", ["gaussian_2d", "draw_heatmap_gaussian", "gaussian_radius"],
                                {"np": __import__("numpy")})
    clip = reference_functions("mmdet3d/models/utils/clip_sigmoid.py", ["clip_sigmoid"])
    xyxy = reference_functions("mmdet3d/core/bbox/structures/utils.py", ["xywhr2xyxyr"])
    coders = _Registry()
    saved = {k: sys.modules.get(k) for k in ("mmcv.cnn", "mmdet3d.core", "mmdet3d.models.utils", "mmdet3d.ops.iou3d",
                                               "mmdet3d.ops.iou3d.iou3d_utils", "mmdet.core", "mmdet.core.bbox", "mmdet.core.bbox.builder",
                                               "mmdet3d.models.dense_heads")}
    stub = types.ModuleType("mmcv.cnn")
    stub.__dict__.update(cnn.__dict__)
    stub.ConvModule, stub.build_conv_layer = CS._RefConvModule, build_conv_layer
    sys.modules["mmcv.cnn"] = stub
    bld = sys.modules["mmdet3d.models.builder"]
    heads = _Registry()

    def build_loss(cfg):
        c = dict(cfg)
        return _LOSSES[c.pop("type")](**c)

    # CenterHead builds its separate heads through `builder.build_head` when constructed, so these stay on the stub builder
    bld.HEADS, bld.build_loss, bld.build_head = heads, build_loss, heads.build
    sys.modules["mmdet3d.models"].builder = bld

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m

    mod("mmdet3d.core", circle_nms=None, draw_heatmap_gaussian=gauss["draw_heatmap_gaussian"], gaussian_radius=gauss["gaussian_radius"],
        xywhr2xyxyr=xyxy["xywhr2xyxyr"])
    mod("mmdet3d.models.utils", clip_sigmoid=clip["clip_sigmoid"])
    mod("mmdet3d.ops.iou3d")
    mod("mmdet3d.ops.iou3d.iou3d_utils", nms_gpu=IO.nms_gpu)
    mod("mmdet.core", build_bbox_coder=coders.build, multi_apply=_multi_apply)
    mod("mmdet.core.bbox", BaseBBoxCoder=object)
    mod("mmdet.core.bbox.builder", BBOX_CODERS=coders)
    pkg = types.ModuleType("mmdet3d.models.dense_heads")
    pkg.__path__ = [os.path.join(REF_ROOT, "mmdet3d/models/dense_heads")]
    sys.modules["mmdet3d.models.dense_heads"] = pkg
    try:
        import importlib.util
        spec = importlib.util.spec_from_file_location("_ref_centerpoint_bbox_coders",
                                                      os.path.join(REF_ROOT, "mmdet3d/core/bbox/coders/centerpoint_bbox_coders.py"))
        coder_mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(coder_mod)
        cp = importlib.import_module("mmdet3d.models.dense_heads.centerpoint_head")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        sys.modules.pop("mmdet3d.models.dense_heads.centerpoint_head", None)
    _HEAD = types.SimpleNamespace(module=cp, CenterHead=cp.CenterHead, CenterPointBBoxCoder=coder_mod.CenterPointBBoxCoder, Boxes=Boxes,
                                  HEADS=heads)
    return _HEAD


def build_center_head(cfg):
    """the reference CenterHead from a config dict (type popped), on the CPU"""
    R = load_center_head()
    c = dict(cfg)
    c.pop("type", None)
    return R.CenterHead(**c)
