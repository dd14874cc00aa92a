"""CPU: the float64 deformable-convolution oracle (oracle/dcn_oracle.py) against torchvision.ops.deform_conv2d in float64 (same offset
layout and bilinear rule; groups through the weight shape) on the test grid, against the grouped conv2d at zero offsets, and the reference's
own DCNSeparateHead (centerpoint_head.py, imported unmodified through oracle/centerpoint_shim.py) against the oracle's restatement of its forward
and against sst_b200's DCNSeparateHead state-dict keys and shapes."""
import copy

import pytest
import torch

from oracle import dcn_oracle as D
from oracle import centerpoint_shim

DCN_CFG = dict(type="DCN", in_channels=64, out_channels=64, kernel_size=3, padding=1, groups=4, bias=False)
# configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py:95-119
SEPARATE_HEAD = dict(type="DCNSeparateHead", init_bias=-2.19, final_kernel=3, dcn_config=DCN_CFG,
                     norm_cfg=dict(type="naiveSyncBN2d", eps=1e-3, momentum=0.01))
COMMON_HEADS = dict(reg=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2))


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("mode", D.OFFSET_MODES)
@pytest.mark.parametrize("case", D.CASES, ids=lambda c: "x".join(map(str, c)))
def test_oracle_matches_torchvision(case, mode):
    tv = pytest.importorskip("torchvision")
    N, C, H, W, O, k, s, p, d, G, dg = case
    x, off, w, gy = (t.double() for t in D.synth_case(case, mode, seed=7 * D.CASES.index(case) + D.OFFSET_MODES.index(mode)))
    xr, orr, wr = (t.clone().requires_grad_(True) for t in (x, off, w))
    yt = tv.ops.deform_conv2d(xr, orr, wr, None, (s, s), (p, p), (d, d))
    yt.backward(gy)
    y = D.deform_conv2d(x, off, w, s, p, d, G, dg)
    gx, goff, gw = D.deform_conv2d_grads(x, off, w, gy, s, p, d, G, dg)
    # a sample exactly at p = -1 lies outside mmcv's open domain, so its offset gradient is 0 there; torchvision's is not
    at_m1 = _at_minus_one(off, k, s, p, d, dg)
    assert (goff[at_m1] == 0).all()
    tv_goff = torch.where(at_m1, 0.0, orr.grad)
    for name, a, b in (("y", y, yt), ("grad_x", gx, xr.grad), ("grad_offset", goff, tv_goff), ("grad_weight", gw, wr.grad)):
        assert _rel(a, b.detach()) <= 1e-12, name


def _at_minus_one(off, k, s, p, d, dg):
    """[N, 2 dg k k, Ho, Wo] mask of the offsets whose sample has p_h = -1 or p_w = -1 exactly"""
    N, _, Ho, Wo = off.shape
    o = off.view(N, dg, k * k, 2, Ho, Wo)
    i = torch.arange(k).repeat_interleave(k).view(k * k, 1, 1)
    j = torch.arange(k).repeat(k).view(k * k, 1, 1)
    ph = torch.arange(Ho).view(1, Ho, 1) * s - p + i * d + o[:, :, :, 0]
    pw = torch.arange(Wo).view(1, 1, Wo) * s - p + j * d + o[:, :, :, 1]
    m = (ph == -1) | (pw == -1)
    return torch.stack([m, m], 3).view(off.shape)


def test_oracle_zero_offsets_is_grouped_conv2d():
    for case in D.CASES:
        N, C, H, W, O, k, s, p, d, G, dg = case
        x, off, w, _ = (t.double() for t in D.synth_case(case, "zero", seed=1))
        ref = torch.nn.functional.conv2d(x, w, None, s, p, d, G)
        assert _rel(D.deform_conv2d(x, off, w, s, p, d, G, dg), ref) <= 1e-12, case


def _ref_head():
    if not centerpoint_shim.available():
        pytest.skip("reference tree not present")
    R = centerpoint_shim.load_centerpoint_head()
    # CenterHead fills in the separate head's keywords per task (centerpoint_head.py:320-327)
    heads = copy.deepcopy(COMMON_HEADS)
    heads.update(dict(heatmap=(3, 2)))
    cfg = copy.deepcopy(SEPARATE_HEAD)
    cfg.update(in_channels=64, heads=heads, num_cls=3)
    cfg.pop("type")
    return R.DCNSeparateHead(**copy.deepcopy(cfg)), cfg


def test_reference_dcn_separate_head_matches_restatement():
    torch.manual_seed(0)
    head, cfg = _ref_head()
    head = head.double().train()
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for name, prm in head.named_parameters():
            prm.copy_(torch.randn(prm.shape, generator=g, dtype=torch.float64) * (0.02 if "conv_offset" in name else 0.1))
    x = torch.randn(2, 64, 13, 11, generator=g, dtype=torch.float64)
    sd = {k: v.clone() for k, v in head.state_dict().items()}
    got = head(x)
    ref = D.dcn_separate_head_forward(x, sd, COMMON_HEADS, training=True, dcn=DCN_CFG)
    assert list(got) == list(ref)
    for k in ref:
        assert _rel(got[k].detach(), ref[k].detach()) <= 1e-12, k


def test_reference_and_sst_b200_heads_share_state_dict_layout():
    head, cfg = _ref_head()
    import sst_b200  # noqa: F401  (registers the head)
    from sst_b200.registry import MODELS
    ours = MODELS.build(dict(copy.deepcopy(cfg), type="DCNSeparateHead"))
    a = {k: tuple(v.shape) for k, v in head.state_dict().items()}
    b = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    assert a == b
    assert list(a) == list(b)
