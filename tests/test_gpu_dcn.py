"""GPU: the native deformable convolution (ops.deform_conv2d, forward and the deterministic backward) and DCNSeparateHead against the
float64 oracle (oracle/dcn_oracle.py) on the CPU.  Tolerance per element, relative to the float64 sum of the absolute values of the
terms that element adds: 1e-5 for y, grad_x and grad_offset, 1e-4 for grad_weight (a sum over every output pixel)."""
import pytest
import torch

from oracle import dcn_oracle as D

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


def _check(name, got, ref, bound, rtol):
    got = got.detach().cpu().double()
    err = (got - ref).abs()
    lim = rtol * bound + 1e-30
    bad = err > lim
    assert not bad.any(), f"{name}: {int(bad.sum())} of {bad.numel()} elements off, worst err / bound " \
                          f"{(err / bound.clamp_min(1e-30)).max().item():.3e}"


def _run(case, x, off, w, gy):
    from sst_b200 import ops
    N, C, H, W, O, k, s, p, d, G, dg = case
    xg, og, wg = (t.to(dev).requires_grad_(True) for t in (x, off, w))
    y = ops.deform_conv2d(xg, og, wg, s, p, d, G, dg)
    y.backward(gy.to(dev))
    ref = D.deform_conv2d(x, off, w, s, p, d, G, dg)
    y_abs = D.deform_conv2d(x.abs(), off, w.abs(), s, p, d, G, dg)
    gx, goff, gw = D.deform_conv2d_grads(x, off, w, gy, s, p, d, G, dg)
    bx, boff, bw = D.deform_conv2d_grads(x, off, w, gy, s, p, d, G, dg, absolute=True)
    _check("y", y, ref, y_abs, 1e-5)
    _check("grad_x", xg.grad, gx, bx, 1e-5)
    _check("grad_offset", og.grad, goff, boff, 1e-5)
    _check("grad_weight", wg.grad, gw, bw, 1e-4)
    return xg, og, wg, y


@pytest.mark.parametrize("mode", D.OFFSET_MODES)
@pytest.mark.parametrize("case", D.CASES, ids=lambda c: "x".join(map(str, c)))
def test_dcn_matches_oracle(case, mode):
    _run(case, *D.synth_case(case, mode, seed=3 * D.CASES.index(case) + D.OFFSET_MODES.index(mode)))


@pytest.mark.parametrize("mode", ("normal", "zero"))
def test_dcn_centerhead_shape(mode):
    case = (1, 64, 468, 468, 64, 3, 1, 1, 1, 4, 1)
    _run(case, *D.synth_case(case, mode, seed=11))


def test_dcn_zero_offsets_is_grouped_conv():
    case = (2, 12, 10, 9, 8, 3, 1, 1, 1, 4, 1)
    x, off, w, gy = D.synth_case(case, "zero", seed=3)
    from sst_b200 import ops
    y = ops.deform_conv2d(x.to(dev), off.to(dev), w.to(dev), 1, 1, 1, 4, 1).cpu().double()
    ref = torch.nn.functional.conv2d(x.double(), w.double(), None, 1, 1, 1, 4)
    assert (y - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


def test_dcn_backward_is_deterministic():
    from sst_b200 import ops
    case = (2, 64, 60, 52, 64, 3, 1, 1, 1, 4, 1)
    x, off, w, gy = (t.to(dev) for t in D.synth_case(case, "normal", seed=5))
    geom = [2, 64, 60, 52, 64, 3, 3, 1, 1, 1, 1, 1, 1, 4, 1]
    a = ops.deform_conv2d_backward(x, off, w, gy, geom)
    b = ops.deform_conv2d_backward(x, off, w, gy, geom)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    y1 = ops.deform_conv2d(x, off, w, 1, 1, 1, 4, 1)
    assert torch.equal(y1, ops.deform_conv2d(x, off, w, 1, 1, 1, 4, 1))


def test_dcn_errors():
    from sst_b200 import ops
    from sst_b200._lib import SSTB200Error
    x, off, w, _ = D.synth_case((1, 8, 9, 11, 8, 3, 1, 1, 1, 1, 1), "normal")
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(x, off, w, 1, 1)                                               # CPU
    xg, og, wg = x.to(dev), off.to(dev), w.to(dev)
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg.half(), og.half(), wg.half(), 1, 1)                          # fp16
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg, og[:, :10], wg, 1, 1)                                       # offset channels
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg, og, wg, 1, 0)                                               # offset spatial size
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg, og, wg[:, :3], 1, 1, groups=2)                              # weight vs groups
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg, og, wg, 1, 1, bias=True)
    with pytest.raises(SSTB200Error):
        ops.deform_conv2d(xg[0], og, wg, 1, 1)                                            # not 4-d


def test_dcn_module_pack_and_old_state_dict():
    from sst_b200.dcn_modules import DeformConv2dPack
    m = DeformConv2dPack(8, 12, 3, padding=1, deformable_groups=2).to(dev)
    assert m.deform_groups == 2 and m.conv_offset.weight.shape == (36, 8, 3, 3)
    x = torch.randn(2, 8, 9, 7, device=dev)
    assert m(x).shape == (2, 12, 9, 7)
    # a version-1 DeformConvPack checkpoint names the offset conv `<prefix>_offset`; loading renames it to conv_offset
    sd = {"weight": m.weight.detach().cpu(), "_offset.weight": torch.randn(36, 8, 3, 3), "_offset.bias": torch.randn(36)}
    m2 = DeformConv2dPack(8, 12, 3, padding=1, deformable_groups=2)
    m2.load_state_dict(sd)
    assert torch.equal(m2.conv_offset.weight, sd["_offset.weight"]) and torch.equal(m2.conv_offset.bias, sd["_offset.bias"])


def test_dcn_separate_head_matches_oracle():
    """DCNSeparateHead (configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py's separate_head, 3-class task) on a 2 x 64 x 96 x 80 map in
    training mode, against the float64 oracle head (dense convs in float64 on the CPU; TF32 off on the GPU).
    Outputs are compared per element.  The gradients of x and of both DCNs (weight, conv_offset) are compared per element too, by running
    the oracle's DCN backward from the gradient the GPU head delivers at each DCN's output: a ReLU pre-activation within fp32 rounding of 0
    flips its mask between fp32 and float64, which moves whole gradient terms, so the dense layers' gradients, upstream of those masks,
    are compared in relative L2 norm."""
    from sst_b200.registry import MODELS
    heads = dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2), heatmap=(3, 2))
    dcn = dict(type="DCN", in_channels=64, out_channels=64, kernel_size=3, padding=1, groups=4, bias=False)
    cfg = dict(type="DCNSeparateHead", init_bias=-2.19, final_kernel=3, dcn_config=dcn,
               norm_cfg=dict(type="naiveSyncBN2d", eps=1e-3, momentum=0.01), in_channels=64, heads=heads, num_cls=3)
    torch.manual_seed(0)
    head = MODELS.build(cfg)
    head.init_weights()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in head.named_parameters():
            # offsets of 0.3 .. 0.7 pixels plus a small input-dependent part: every sample stays clear of integer positions, where
            # grad_offset jumps and the fp32 and float64 offset convolutions could pick different corners
            if name.endswith("conv_offset.weight"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.002)
            elif name.endswith("conv_offset.bias"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.4 + 0.3)
    head = head.to(dev).train()
    x = torch.randn(2, 64, 96, 80, generator=g)
    params = dict(head.named_parameters())
    sd = {k: v.detach().cpu().double().requires_grad_(k in params) for k, v in head.state_dict().items()}
    xo = x.double().requires_grad_(True)
    ref = D.dcn_separate_head_forward(xo, sd, {k: v for k, v in heads.items() if k != "heatmap"}, training=True, dcn=dcn)
    probes = {k: torch.randn(v.shape, generator=g, dtype=torch.float64) for k, v in ref.items()}
    sum((ref[k] * probes[k]).sum() for k in ref).backward()
    feats = {}

    def keep(name):
        def hook(module, inputs, output):
            output.retain_grad()
            feats[name] = output
        return hook

    hooks = [getattr(head, n).register_forward_hook(keep(n)) for n in ("feature_adapt_cls", "feature_adapt_reg")]
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        xg = x.to(dev).requires_grad_(True)
        out = head(xg)
        sum((out[k] * probes[k].float().to(dev)).sum() for k in out).backward()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
        for h in hooks:
            h.remove()
    assert set(out) == set(ref)
    rel = lambda a, b: (a.detach().cpu().double() - b).abs().max().item() / b.abs().max().clamp_min(1e-30).item()
    for k in ref:
        assert rel(out[k], ref[k].detach()) < 1e-4, k
    # the DCN layers' backward from the GPU head's own gradients at their outputs
    sd2 = {k: v.detach().clone().requires_grad_(k in params) for k, v in sd.items()}
    x2 = x.double().requires_grad_(True)
    for n in ("feature_adapt_cls", "feature_adapt_reg"):
        y = D.dcn_pack_forward(x2, sd2, n + ".", stride=1, padding=1, dilation=1, groups=4, deform_groups=1)
        y.backward(feats[n].grad.cpu().double())
    assert rel(xg.grad, x2.grad) < 1e-4
    for name, p in head.named_parameters():
        if name.startswith("feature_adapt"):
            assert rel(p.grad, sd2[name].grad) < 1e-4, name
        else:
            l2 = ((p.grad.cpu().double() - sd[name].grad).norm() / sd[name].grad.norm()).item()
            assert l2 < 1e-2, (name, l2)
