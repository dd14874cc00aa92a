"""TEST INFRASTRUCTURE ONLY - never imported by the product package.

Imports the reference's own mmdet3d/models/dense_heads/centerpoint_head.py unmodified, on top of oracle/ref_shim.py's stubs, so that its
SeparateHead / DCNSeparateHead can be built on the CPU: mmcv's ConvModule is restated here, 'DCN' is built from the float64 deformable
convolution of oracle/dcn_oracle.py, and the names the file's import line pulls in that the two heads never use (box coding, losses, NMS)
are stubbed while it is imported."""
import importlib
import os
import sys
import types

import torch
import torch.nn as nn

from oracle.ref_shim import REF_ROOT, _Registry, available, load  # noqa: F401  (available: for the tests' skip)




class _RefConvModule(nn.Module):
    """mmcv.cnn.ConvModule (1.3.x) restated as far as centerpoint_head.py uses it: conv -> norm -> activation in that order, children
    `conv`, the norm's abbreviation (`bn`) and `activate`; bias='auto' = a conv bias only without a norm."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias="auto", conv_cfg=None,
                 norm_cfg=None, act_cfg=dict(type="ReLU"), inplace=True, **kwargs):
        super().__init__()
        cnn = sys.modules["mmcv.cnn"]
        with_norm = norm_cfg is not None
        if bias == "auto":
            bias = not with_norm
        self.conv = cnn.build_conv_layer(conv_cfg, in_channels, out_channels, kernel_size, stride=stride, padding=padding,
                                         dilation=dilation, groups=groups, bias=bias)
        self.norm_name = None
        if with_norm:
            self.norm_name, norm = cnn.build_norm_layer(norm_cfg, out_channels)
            self.add_module(self.norm_name, norm)
        self.activate = nn.ReLU(inplace=inplace) if act_cfg is not None else None

    def forward(self, x):
        x = self.conv(x)
        if self.norm_name is not None:
            x = getattr(self, self.norm_name)(x)
        return self.activate(x) if self.activate is not None else x


class _OracleDCN(nn.Module):
    """mmcv's DeformConv2dPack ('DCN') over oracle/dcn_oracle.py: parameters `weight` and `conv_offset` (zero-initialised)"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False,
                 im2col_step=32):
        super().__init__()
        assert not bias
        k = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        self.cfg = (stride, padding, dilation, groups, deform_groups)
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, *k).uniform_(-1, 1) / (in_channels * k[0] * k[1]) ** 0.5)
        self.conv_offset = nn.Conv2d(in_channels, deform_groups * 2 * k[0] * k[1], k, stride, padding, dilation, bias=True)
        nn.init.zeros_(self.conv_offset.weight)
        nn.init.zeros_(self.conv_offset.bias)

    def forward(self, x):
        from oracle import dcn_oracle
        return dcn_oracle.DeformConv2dFunction.apply(x, self.conv_offset(x), self.weight, *self.cfg)


_CENTERPOINT = None


def load_centerpoint_head():
    """The reference's own mmdet3d/models/dense_heads/centerpoint_head.py, imported unmodified, with mmcv's ConvModule restated, 'DCN'
    built from the oracle's deformable convolution, and stubs for the names its import line pulls in that SeparateHead / DCNSeparateHead
    never use (box coding, losses, NMS).  The stubs are removed from sys.modules again once the file is imported."""
    global _CENTERPOINT
    if _CENTERPOINT is not None:
        return _CENTERPOINT
    load()
    cnn = sys.modules["mmcv.cnn"]
    dense_build = cnn.build_conv_layer

    def build_conv_layer(cfg, *args, **kwargs):
        c = dict(cfg or dict(type="Conv2d"))
        if c.get("type") == "DCN":
            c.pop("type")
            return _OracleDCN(*args, **kwargs, **c)
        return dense_build(cfg, *args, **kwargs)

    saved = {k: sys.modules.get(k) for k in ("mmcv.cnn", "mmdet3d.core", "mmdet3d.models.utils", "mmdet3d.ops.iou3d",
                                               "mmdet3d.ops.iou3d.iou3d_utils", "mmdet.core", "mmdet3d.models.dense_heads")}
    stub = types.ModuleType("mmcv.cnn")
    stub.__dict__.update(cnn.__dict__)
    stub.ConvModule, stub.build_conv_layer = _RefConvModule, build_conv_layer
    sys.modules["mmcv.cnn"] = stub
    bld = sys.modules["mmdet3d.models.builder"]
    heads = _Registry()
    added = [a for a in ("HEADS", "build_loss", "build_head") if not hasattr(bld, a)]
    bld.HEADS, bld.build_loss, bld.build_head = heads, None, heads.build
    for name, attrs in (("mmdet3d.core", dict(circle_nms=None, draw_heatmap_gaussian=None, gaussian_radius=None, xywhr2xyxyr=None)),
                        ("mmdet3d.models.utils", dict(clip_sigmoid=None)), ("mmdet3d.ops.iou3d", {}),
                        ("mmdet3d.ops.iou3d.iou3d_utils", dict(nms_gpu=None)), ("mmdet.core", dict(build_bbox_coder=None, multi_apply=None))):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    pkg = types.ModuleType("mmdet3d.models.dense_heads")
    pkg.__path__ = [os.path.join(REF_ROOT, "mmdet3d/models/dense_heads")]
    sys.modules["mmdet3d.models.dense_heads"] = pkg
    try:
        cp = importlib.import_module("mmdet3d.models.dense_heads.centerpoint_head")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        sys.modules.pop("mmdet3d.models.dense_heads.centerpoint_head", None)
        for a in added:
            delattr(bld, a)
    _CENTERPOINT = types.SimpleNamespace(module=cp, SeparateHead=cp.SeparateHead, DCNSeparateHead=cp.DCNSeparateHead, HEADS=heads)
    return _CENTERPOINT
