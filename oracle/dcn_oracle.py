"""Float64 restatement of mmcv 1.3.8-1.4.0 deform_conv2d (the 'DCN' of CenterHead's DCNSeparateHead): forward and the three gradients
as explicit formulas, chunked over output rows so that a 1 x 64 x 468 x 468 map fits on the CPU.  Test infrastructure only.

Sampling: p = (integer base) + offset as ONE addition in the offset's dtype (fp32 offsets: the fp32 sum the CUDA path forms), then every
later step in float64.  S = 0 unless -1 < p_h < H and -1 < p_w < W, else the bilinear blend of the corners floor(p), floor(p) + 1, a corner
outside the image counting 0.  grad_offset holds the corners at floor(p) (forward difference at an integer p)."""
import math

import torch
import torch.nn.functional as F

_CHUNK_ELEMS = 1 << 22  # float64 elements of one chunk's sampled columns


def _pair(v):
    return (int(v), int(v)) if isinstance(v, (int, float)) else (int(v[0]), int(v[1]))


def out_size(H, W, kernel, stride, padding, dilation):
    (kh, kw), (sh, sw), (ph, pw), (dh, dw) = _pair(kernel), _pair(stride), _pair(padding), _pair(dilation)
    return (H + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1


def _sample(x, offset, r0, r1, kh, kw, stride, padding, dilation, dg):
    """Output rows [r0, r1): per corner (lists of 4, [N, dg, K, R, Wo]) the flat pixel index, the weight (0 outside the image) and the
    inside-the-image mask; then the fractions lh, lw and the sample's validity."""
    N, C, H, W = x.shape
    Wo = offset.shape[3]
    K, R = kh * kw, r1 - r0
    (sh, sw), (ph, pw), (dh, dw) = stride, padding, dilation
    off = offset[:, :, r0:r1].reshape(N, dg, K, 2, R, Wo)
    ki = torch.arange(kh).repeat_interleave(kw).view(K, 1, 1)
    kj = torch.arange(kw).repeat(kh).view(K, 1, 1)
    base_h = torch.arange(r0, r1).view(1, R, 1) * sh - ph + ki * dh
    base_w = torch.arange(Wo).view(1, 1, Wo) * sw - pw + kj * dw
    p_h = (base_h.to(off.dtype) + off[:, :, :, 0]).double()
    p_w = (base_w.to(off.dtype) + off[:, :, :, 1]).double()
    valid = (p_h > -1) & (p_w > -1) & (p_h < H) & (p_w < W)
    h0, w0 = torch.floor(p_h), torch.floor(p_w)
    lh, lw = torch.where(valid, p_h - h0, 0.0), torch.where(valid, p_w - w0, 0.0)
    hh, hw = 1 - lh, 1 - lw
    idx, wts, masks = [], [], []
    for dy, dx, wq in ((0, 0, hh * hw), (0, 1, hh * lw), (1, 0, lh * hw), (1, 1, lh * lw)):
        h, w = h0.long() + dy, w0.long() + dx
        m = valid & (h >= 0) & (w >= 0) & (h < H) & (w < W)
        idx.append(torch.where(m, h * W + w, 0))
        wts.append(torch.where(m, wq, 0.0))
        masks.append(m)
    return idx, wts, masks, lh, lw, valid


def _gather(xd, idx):
    """xd [N, dg, Cd, HW], idx [N, dg, K, R, Wo] -> [N, dg, Cd, K, R, Wo]"""
    N, dg, Cd, _ = xd.shape
    shp = idx.shape
    flat = idx.reshape(N, dg, 1, -1).expand(N, dg, Cd, -1)
    return torch.gather(xd, 3, flat).view(N, dg, Cd, *shp[2:])


def _rows_per_chunk(C, K, Wo):
    return max(1, _CHUNK_ELEMS // max(1, C * K * Wo))


def _geom(x, offset, weight, stride, padding, dilation, groups, deform_groups):
    N, C, H, W = x.shape
    O, Cg, kh, kw = weight.shape
    assert C == Cg * groups and O % groups == 0 and C % deform_groups == 0
    Ho, Wo = out_size(H, W, (kh, kw), stride, padding, dilation)
    assert offset.shape == (N, 2 * deform_groups * kh * kw, Ho, Wo), offset.shape
    return N, C, H, W, O, Cg, kh, kw, Ho, Wo


def deform_conv2d(x, offset, weight, stride=1, padding=0, dilation=1, groups=1, deform_groups=1):
    """float64 y [N, Cout, Ho, Wo]"""
    stride, padding, dilation = _pair(stride), _pair(padding), _pair(dilation)
    N, C, H, W, O, Cg, kh, kw, Ho, Wo = _geom(x, offset, weight, stride, padding, dilation, groups, deform_groups)
    K, dg = kh * kw, deform_groups
    xd = x.double().reshape(N, dg, C // dg, H * W)
    w = weight.double().reshape(groups, O // groups, Cg * K)
    y = torch.empty(N, O, Ho, Wo, dtype=torch.float64)
    step = _rows_per_chunk(C, K, Wo)
    for r0 in range(0, Ho, step):
        r1 = min(Ho, r0 + step)
        idx, wts, _, _, _, _ = _sample(x, offset, r0, r1, kh, kw, stride, padding, dilation, dg)
        col = sum(_gather(xd, i) * wq[:, :, None] for i, wq in zip(idx, wts))          # [N, dg, Cd, K, R, Wo]
        col = col.reshape(N, groups, Cg * K, (r1 - r0) * Wo)
        y[:, :, r0:r1] = torch.einsum("gor,ngrp->ngop", w, col).reshape(N, O, r1 - r0, Wo)
    return y


def deform_conv2d_grads(x, offset, weight, grad_y, stride=1, padding=0, dilation=1, groups=1, deform_groups=1, absolute=False):
    """float64 (grad_x, grad_offset, grad_weight) for the upstream gradient grad_y.  absolute=True: instead, per element the sum of the
    absolute values of the terms it adds (|x|, |W|, |grad_y| and, for grad_offset, |v| in place of the corner differences)"""
    stride, padding, dilation = _pair(stride), _pair(padding), _pair(dilation)
    if absolute:
        x, weight, grad_y = x.double().abs(), weight.double().abs(), grad_y.double().abs()
    N, C, H, W, O, Cg, kh, kw, Ho, Wo = _geom(x, offset, weight, stride, padding, dilation, groups, deform_groups)
    K, dg, Cd = kh * kw, deform_groups, C // deform_groups
    xd = x.double().reshape(N, dg, Cd, H * W)
    w = weight.double().reshape(groups, O // groups, Cg * K)
    gy = grad_y.double().reshape(N, groups, O // groups, Ho, Wo)
    gx = torch.zeros(N, dg, Cd, H * W, dtype=torch.float64)
    goff = torch.empty(N, dg, K, 2, Ho, Wo, dtype=torch.float64)
    gw = torch.zeros(groups, O // groups, Cg * K, dtype=torch.float64)
    step = _rows_per_chunk(C, K, Wo)
    for r0 in range(0, Ho, step):
        r1 = min(Ho, r0 + step)
        R = r1 - r0
        idx, wts, masks, lh, lw, valid = _sample(x, offset, r0, r1, kh, kw, stride, padding, dilation, dg)
        v = [_gather(xd, i) * m[:, :, None] for i, m in zip(idx, masks)]                  # corner values, 0 outside the image
        col = sum(vq * wq[:, :, None] for vq, wq in zip(v, wts))                           # [N, dg, Cd, K, R, Wo]
        g_r = gy[:, :, :, r0:r1].reshape(N, groups, O // groups, R * Wo)
        gw += torch.einsum("ngop,ngrp->gor", g_r, col.reshape(N, groups, Cg * K, R * Wo))
        gcol = torch.einsum("gor,ngop->ngrp", w, g_r).reshape(N, dg, Cd, K, R, Wo)
        hh, hw = 1 - lh, 1 - lw
        sg = 1 if absolute else -1
        dsh = hw[:, :, None] * (v[2] + sg * v[0]) + lw[:, :, None] * (v[3] + sg * v[1])
        dsw = hh[:, :, None] * (v[1] + sg * v[0]) + lh[:, :, None] * (v[3] + sg * v[2])
        goff[:, :, :, 0, r0:r1] = torch.where(valid, (gcol * dsh).sum(2), 0.0)
        goff[:, :, :, 1, r0:r1] = torch.where(valid, (gcol * dsw).sum(2), 0.0)
        for i, wq in zip(idx, wts):
            src = (gcol * wq[:, :, None]).reshape(N, dg, Cd, -1)
            gx.scatter_add_(3, i.reshape(N, dg, 1, -1).expand(N, dg, Cd, -1), src)
    return gx.reshape(N, C, H, W), goff.reshape(N, 2 * dg * K, Ho, Wo), gw.reshape(O, Cg, kh, kw)



class DeformConv2dFunction(torch.autograd.Function):
    """autograd over the explicit formulas above (float64 outputs and gradients)"""

    @staticmethod
    def forward(ctx, x, offset, weight, stride, padding, dilation, groups, deform_groups):
        ctx.save_for_backward(x, offset, weight)
        ctx.cfg = (stride, padding, dilation, groups, deform_groups)
        return deform_conv2d(x, offset, weight, *ctx.cfg)

    @staticmethod
    def backward(ctx, grad_y):
        x, offset, weight = ctx.saved_tensors
        gx, goff, gw = deform_conv2d_grads(x, offset, weight, grad_y, *ctx.cfg)
        return gx.to(x.dtype), goff.to(offset.dtype), gw.to(weight.dtype), None, None, None, None, None


def dcn_pack_forward(x, sd, prefix, stride=1, padding=1, dilation=1, groups=1, deform_groups=1):
    """DeformConv2dPack: offset = conv2d(x, conv_offset) (same kernel / stride / padding / dilation), then deform_conv2d"""
    w = sd[prefix + "weight"]
    offset = F.conv2d(x, sd[prefix + "conv_offset.weight"], sd[prefix + "conv_offset.bias"], stride, padding, dilation)
    return DeformConv2dFunction.apply(x, offset, w, stride, padding, dilation, groups, deform_groups)


def dcn_separate_head_forward(x, sd, heads, training, head_eps=1e-3, task_eps=1e-5, momentum=0.01, dcn=None):
    """Restatement of DCNSeparateHead.forward (centerpoint_head.py:208-238) over a state dict of float64 tensors (autograd-able):
    feature_adapt_{cls,reg} = DCN; cls_head = conv3x3 (no bias) + BN(head_eps) + ReLU, conv3x3 + bias; task_head.<head> = (num_conv - 1) x
    [conv(final_kernel, no bias) + BN2d(task_eps) + ReLU] + conv(final_kernel) + bias.  heads: {name: (classes, num_conv)} without
    'heatmap'; BN uses batch statistics when training.  dcn: DCN keywords (kernel_size, padding, groups, ...)."""
    dcn = dict(dcn or {})
    kd = dict(stride=dcn.get("stride", 1), padding=dcn.get("padding", 0), dilation=dcn.get("dilation", 1), groups=dcn.get("groups", 1),
              deform_groups=dcn.get("deform_groups", 1))

    def bn(t, p, eps):
        return F.batch_norm(t, sd[p + "running_mean"].clone(), sd[p + "running_var"].clone(), sd[p + "weight"], sd[p + "bias"], training,
                            momentum, eps)

    def conv(t, p, bias):
        k = sd[p + "weight"].shape[-1]
        return F.conv2d(t, sd[p + "weight"], sd[p + "bias"] if bias else None, 1, k // 2)

    center = dcn_pack_forward(x, sd, "feature_adapt_cls.", **kd)
    reg = dcn_pack_forward(x, sd, "feature_adapt_reg.", **kd)
    h = F.relu(bn(conv(center, "cls_head.0.conv.", False), "cls_head.0.bn.", head_eps))
    ret = {}
    for name, (_, num_conv) in heads.items():
        t = reg
        for i in range(num_conv - 1):
            t = F.relu(bn(conv(t, f"task_head.{name}.{i}.conv.", False), f"task_head.{name}.{i}.bn.", task_eps))
        ret[name] = conv(t, f"task_head.{name}.{num_conv - 1}.", True)
    ret["heatmap"] = conv(h, "cls_head.1.", True)
    return ret


# test grid: (N, Cin, H, W, Cout, kernel, stride, padding, dilation, groups, deform_groups)
CASES = [
    (1, 8, 9, 11, 8, 3, 1, 1, 1, 1, 1),
    (2, 8, 7, 7, 12, 3, 2, 1, 1, 2, 2),
    (1, 16, 13, 9, 16, 3, 1, 2, 2, 4, 4),
    (1, 4, 5, 6, 4, 5, 1, 2, 1, 1, 1),
    (3, 6, 6, 5, 10, 1, 1, 0, 1, 2, 1),
    (1, 4, 1, 1, 4, 1, 1, 0, 1, 4, 2),
    (1, 12, 9, 9, 20, 3, 2, 0, 1, 4, 2),
    (2, 5, 8, 7, 7, 3, 1, 1, 2, 1, 1),
    (1, 8, 3, 3, 8, 5, 2, 2, 1, 2, 4),
    (1, 64, 12, 10, 64, 3, 1, 1, 1, 4, 1),
    (1, 128, 6, 6, 96, 3, 1, 1, 1, 1, 1),
    (1, 32, 5, 7, 64, 3, 1, 1, 1, 2, 1),
    (2, 16, 40, 40, 16, 3, 1, 1, 1, 1, 1),
]
OFFSET_MODES = ("normal", "large", "integer")


def synth_case(case, mode, seed=0, dtype=torch.float32):
    """x, offset, weight, grad_y of one grid case.  Offsets: normal = N(0, 1.5^2) pixels; large = uniform in +-2 max(H, W); integer =
    whole pixels in [-(H + 2), H + 2], so samples land exactly on pixels and exactly at -1 and H."""
    N, C, H, W, O, k, s, p, d, G, dg = case
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = out_size(H, W, k, s, p, d)
    x = torch.randn(N, C, H, W, generator=g)
    oshape = (N, 2 * dg * k * k, Ho, Wo)
    if mode == "normal":
        off = torch.randn(oshape, generator=g) * 1.5
    elif mode == "large":
        off = (torch.rand(oshape, generator=g) * 2 - 1) * 2 * max(H, W)
    elif mode == "integer":
        off = torch.randint(-(max(H, W) + 2), max(H, W) + 3, oshape, generator=g).float()
    elif mode == "zero":
        off = torch.zeros(oshape)
    else:
        raise ValueError(mode)
    w = torch.randn(O, C // G, k, k, generator=g) / math.sqrt(C // G * k * k)
    gy = torch.randn(N, O, Ho, Wo, generator=g)
    return x.to(dtype), off.to(dtype), w.to(dtype), gy.to(dtype)
