"""CenterHead's deformable-convolution head on libsstb200: mmcv 1.3.8-1.4.0 DeformConv2d / DeformConv2dPack ('DCN') over
ops.deform_conv2d, a dense build_conv_layer, mmcv's ConvModule as far as the head uses it, and SeparateHead / DCNSeparateHead
(mmdet3d/models/dense_heads/centerpoint_head.py:17-238) with the reference's constructor keywords and state-dict keys."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from . import ops
from . import spconv_modules
from .registry import MODELS, Registry


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


class DeformConv2d(nn.Module):
    """mmcv.ops.DeformConv2d: parameter `weight` [Cout, Cin / groups, kh, kw], no bias (bias=True raises, as in mmcv).  The old keyword
    `deformable_groups` is accepted for `deform_groups`."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, bias=False,
                 im2col_step=32, deformable_groups=None):
        super().__init__()
        if deformable_groups is not None:
            deform_groups = deformable_groups
        assert not bias, f"bias={bias} is not supported in DeformConv2d."
        assert in_channels % groups == 0, f"in_channels {in_channels} cannot be divisible by groups {groups}"
        assert out_channels % groups == 0, f"out_channels {out_channels} cannot be divisible by groups {groups}"
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = _pair(kernel_size), _pair(stride), _pair(padding), _pair(dilation)
        self.groups, self.deform_groups, self.im2col_step = groups, deform_groups, im2col_step
        self.transposed, self.output_padding = False, _pair(0)
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()

    def reset_parameters(self):
        n = self.in_channels * self.kernel_size[0] * self.kernel_size[1]
        stdv = 1.0 / math.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)

    def forward(self, x, offset):
        # mmcv pads an input smaller than the kernel on the bottom / right and crops the output back
        pad_h, pad_w = max(self.kernel_size[0] - x.size(2), 0), max(self.kernel_size[1] - x.size(3), 0)
        if pad_h or pad_w:
            x = F.pad(x, (0, pad_w, 0, pad_h), "constant", 0).contiguous()
            offset = F.pad(offset, (0, pad_w, 0, pad_h), "constant", 0).contiguous()
        out = ops.deform_conv2d(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups, self.deform_groups, False,
                                self.im2col_step)
        if pad_h or pad_w:
            out = out[:, :, :out.size(2) - pad_h, :out.size(3) - pad_w].contiguous()
        return out


class DeformConv2dPack(DeformConv2d):
    """mmcv.ops.DeformConv2dPack ('DCN'): the offsets come from conv_offset = Conv2d(Cin, dg * 2 * kh * kw, same kernel / stride / padding
    / dilation, bias=True), zero-initialised.  State dicts of version < 2 name it `<prefix>_offset`; loading renames it."""
    _version = 2

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deform_groups * 2 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=self.stride, padding=self.padding, dilation=self.dilation,
                                     bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        return super().forward(x, self.conv_offset(x))

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        version = local_metadata.get("version", None)
        if version is None or version < 2:
            for p in ("weight", "bias"):
                old = prefix[:-1] + "_offset." + p
                if prefix + "conv_offset." + p not in state_dict and old in state_dict:
                    state_dict[prefix + "conv_offset." + p] = state_dict.pop(old)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)


CONV_LAYERS = Registry("conv layer")
CONV_LAYERS.register_module("Conv2d", module=nn.Conv2d)
CONV_LAYERS.register_module("Conv", module=nn.Conv2d)
CONV_LAYERS.register_module("DCN", module=DeformConv2dPack)


def build_conv_layer(cfg, *args, **kwargs):
    """mmcv.cnn.build_conv_layer: None / 'Conv2d' / 'Conv' -> nn.Conv2d, 'DCN' -> DeformConv2dPack; the sparse types go to
    spconv_modules.build_conv_layer"""
    cfg = dict(type="Conv2d") if cfg is None else dict(cfg)
    t = cfg.pop("type")
    if t in CONV_LAYERS:
        return CONV_LAYERS.get(t)(*args, **kwargs, **cfg)
    return spconv_modules.build_conv_layer(dict(cfg, type=t), *args, **kwargs)


class ConvModule(nn.Module):
    """mmcv.cnn.ConvModule as the head builds it: conv -> norm -> ReLU, children `conv`, the norm's abbreviation (`bn`) and `activate`;
    bias='auto' means a conv bias only without a norm."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias="auto", conv_cfg=None,
                 norm_cfg=None, act_cfg=dict(type="ReLU"), inplace=True):
        super().__init__()
        with_norm = norm_cfg is not None
        if bias == "auto":
            bias = not with_norm
        self.conv = build_conv_layer(conv_cfg, in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                                     groups=groups, bias=bias)
        self.norm_name = None
        if with_norm:
            self.norm_name, norm = ops.build_norm_layer(norm_cfg, out_channels)
            self.add_module(self.norm_name, norm)
        self.activate = None
        if act_cfg is not None:
            assert act_cfg["type"] == "ReLU", act_cfg
            self.activate = nn.ReLU(inplace=inplace)

    def forward(self, x):
        x = self.conv(x)
        if self.norm_name is not None:
            x = getattr(self, self.norm_name)(x)
        if self.activate is not None:
            x = self.activate(x)
        return x


def _kaiming_conv2d(module):
    """mmcv's init_cfg dict(type='Kaiming', layer='Conv2d'): kaiming_normal_(fan_out, relu) and zero bias on every nn.Conv2d"""
    for m in module.modules():
        if type(m) is nn.Conv2d:
            nn.init.kaiming_normal_(m.weight, a=0, mode="fan_out", nonlinearity="relu")
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)


@MODELS.register_module()
class SeparateHead(nn.Module):
    """centerpoint_head.py:17-120.  heads = {name: (classes, num_conv)}: per head (num_conv - 1) ConvModules (final_kernel, no conv bias
    under a norm) and a final conv with a bias; forward -> {name: [B, classes, H, W]}."""

    def __init__(self, in_channels, heads, head_conv=64, final_kernel=1, init_bias=-2.19, conv_cfg=dict(type="Conv2d"),
                 norm_cfg=dict(type="BN2d"), bias="auto", init_cfg=None, **kwargs):
        assert init_cfg is None, "To prevent abnormal initialization behavior, init_cfg is not allowed to be set"
        super().__init__()
        self.heads = heads
        self.init_bias = init_bias
        for head in self.heads:
            classes, num_conv = self.heads[head]
            conv_layers = []
            c_in = in_channels
            for _ in range(num_conv - 1):
                conv_layers.append(ConvModule(c_in, head_conv, kernel_size=final_kernel, stride=1, padding=final_kernel // 2, bias=bias,
                                              conv_cfg=conv_cfg, norm_cfg=norm_cfg))
                c_in = head_conv
            conv_layers.append(build_conv_layer(conv_cfg, head_conv, classes, kernel_size=final_kernel, stride=1,
                                                padding=final_kernel // 2, bias=True))
            self.__setattr__(head, nn.Sequential(*conv_layers))

    def init_weights(self):
        _kaiming_conv2d(self)
        for head in self.heads:
            if head == "heatmap":
                self.__getattr__(head)[-1].bias.data.fill_(self.init_bias)

    def forward(self, x):
        return {head: self.__getattr__(head)(x) for head in self.heads}


@MODELS.register_module()
class DCNSeparateHead(nn.Module):
    """centerpoint_head.py:123-238: feature_adapt_cls / feature_adapt_reg = build_conv_layer(dcn_config); cls_head = ConvModule(3x3,
    norm_cfg) + conv 3x3 (bias='auto' reaches nn.Conv2d as a truthy bias); task_head = SeparateHead(in_channels, heads, head_conv,
    final_kernel, bias) with the default BN2d, not norm_cfg.  'heatmap' is popped from `heads` (the caller's dict, as there)."""

    def __init__(self, in_channels, num_cls, heads, dcn_config, head_conv=64, final_kernel=1, init_bias=-2.19,
                 conv_cfg=dict(type="Conv2d"), norm_cfg=dict(type="BN2d"), bias="auto", init_cfg=None, **kwargs):
        assert init_cfg is None, "To prevent abnormal initialization behavior, init_cfg is not allowed to be set"
        super().__init__()
        if "heatmap" in heads:
            heads.pop("heatmap")
        self.feature_adapt_cls = build_conv_layer(dcn_config)
        self.feature_adapt_reg = build_conv_layer(dcn_config)
        self.cls_head = nn.Sequential(
            ConvModule(in_channels, head_conv, kernel_size=3, padding=1, conv_cfg=conv_cfg, bias=bias, norm_cfg=norm_cfg),
            build_conv_layer(conv_cfg, head_conv, num_cls, kernel_size=3, stride=1, padding=1, bias=bias))
        self.init_bias = init_bias
        self.task_head = SeparateHead(in_channels, heads, head_conv=head_conv, final_kernel=final_kernel, bias=bias)

    def init_weights(self):
        _kaiming_conv2d(self)
        self.cls_head[-1].bias.data.fill_(self.init_bias)

    def forward(self, x):
        center_feat = self.feature_adapt_cls(x)
        reg_feat = self.feature_adapt_reg(x)
        ret = self.task_head(reg_feat)
        ret["heatmap"] = self.cls_head(center_feat)
        return ret
