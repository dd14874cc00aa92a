"""GPU parity: window partition / bucketing (B1-B7) and the SRA encoder stack (A1-A4) vs the CPU oracle."""
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]
DROP_TRAIN = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
              2: {'max_tokens': 100, 'drop_range': (60, 100000)}}
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}


def _voxels(seeds, P, C=128, dense=False):
    cs = []
    for b, s in enumerate(seeds):
        p = O.synth_frame(s, P)
        if dense:  # squeeze the sweep so that windows overflow max_tokens (exercises the drop path)
            p[:, :2] *= 0.25
        c = torch.unique(O.dynamic_voxelize(p, VS, RNG), dim=0)
        cs.append(torch.nn.functional.pad(c, (1, 0), value=b))
    coors = torch.cat(cs).int()
    g = torch.Generator().manual_seed(sum(seeds))
    return torch.randn(coors.shape[0], C, generator=g), coors


def _check_info(info_g, info_o):
    for k in ("voxel_coors", "voxel_keep_inds"):
        assert torch.equal(info_g[k].cpu(), info_o[k]), k
    for i in range(2):
        for k in (f"batch_win_inds_shift{i}", f"coors_in_win_shift{i}", f"voxel_drop_level_shift{i}"):
            assert torch.equal(info_g[k].cpu(), info_o[k]), k
        dg, do = info_g[f"flat2win_inds_shift{i}"], info_o[f"flat2win_inds_shift{i}"]
        assert set(k for k in dg if not isinstance(k, str)) == set(k for k in do if not isinstance(k, str))
        for dl in do:
            if isinstance(dl, str):
                continue
            assert torch.equal(dg[dl][0].cpu(), do[dl][0]), (i, dl)
            assert torch.equal(dg[dl][1][0].cpu(), do[dl][1][0]), (i, dl)
            torch.testing.assert_close(info_g[f"pos_dict_shift{i}"][dl].cpu(), info_o[f"pos_dict_shift{i}"][dl],
                                       rtol=0, atol=1e-6)
            assert torch.equal(info_g[f"key_mask_shift{i}"][dl].cpu(), info_o[f"key_mask_shift{i}"][dl])


@pytest.mark.parametrize("seeds,P", [((1000,), 150000), ((3, 4, 5), 20000), ((9,), 300)])
def test_input_layer_eval_bitexact(cuda, seeds, P):
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels(seeds, P)
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    info_g = il(feats.to(cuda), coors.to(cuda), len(seeds))
    info_o = O.input_layer_v2(feats, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    _check_info(info_g, info_o)
    assert torch.equal(info_g["voxel_feats"].cpu(), info_o["voxel_feats"])


def test_input_layer_train_drop_and_shuffle(cuda):
    """Training drop_info (windows > 100 tokens lose voxels) with an injected shuffle: same survivors, same
    levels, same slots as the oracle (canonical stable inner order, SURVEY 8c / F7)."""
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels((11, 12), 150000, C=16, dense=True)
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=True, mute=True).train()
    torch.manual_seed(5)
    info_g = il(feats.to(cuda), coors.to(cuda), 2)
    sh = info_g["shuffle_inds"].cpu()
    info_o = O.input_layer_v2(feats, coors, DROP_TRAIN, (12, 12, 1), (468, 468, 1), shuffle_inds=sh)
    assert info_o["voxel_coors"].shape[0] < coors.shape[0], "test must actually drop voxels"
    _check_info(info_g, info_o)


def test_window_ops_compat(cuda):
    """Standalone op-surface functions (get_window_coors, make_continuous_inds, flat2window/window2flat)."""
    from sst_b200 import ops
    feats, coors = _voxels((21,), 20000, C=8)
    c = coors.long()
    for shift in (False, True):
        rw, rc = O.get_window_coors(c, (468, 468, 1), (12, 12, 1), shift)
        gw, gc = ops.get_window_coors(c.to(cuda), (468, 468, 1), (12, 12, 1), shift)
        assert torch.equal(gw.cpu(), rw) and torch.equal(gc.cpu(), rc)
    assert torch.equal(ops.make_continuous_inds(rw.to(cuda)).cpu(), O.make_continuous_inds(rw))
    keep, lvl = O.drop_single_shift(rw, DROP_TEST)
    d_o = O.get_flat2win_inds(rw, lvl, DROP_TEST)
    d_g = ops.get_flat2win_inds_v2(rw.to(cuda), lvl.to(cuda), DROP_TEST)
    f3_o = O.flat2window(feats, d_o)
    f3_g = ops.flat2window_v2(feats.to(cuda), d_g)
    for dl in f3_o:
        assert torch.equal(f3_g[dl].cpu(), f3_o[dl])
    assert torch.equal(ops.window2flat_v2(f3_g, d_g).cpu(), feats)


def _sst_pair(d, h, ff, blocks, layer_cfg=None, act="gelu", in_channel=None):
    from sst_b200.sst_modules import SSTv2
    torch.manual_seed(0)
    m = SSTv2(d_model=[d] * blocks, nhead=[h] * blocks, num_blocks=blocks, dim_feedforward=[ff] * blocks,
              output_shape=[468, 468], num_attached_conv=0, to_bev=False, activation=act, layer_cfg=layer_cfg or {},
              in_channel=in_channel).eval()
    # non-trivial norms / biases so that every term is exercised
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
            if n_.endswith("tau"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.5 + 0.05)
        for n_, b in m.named_buffers():
            if "running_mean" in n_:
                b.copy_(torch.randn(b.shape, generator=g) * 0.3)
            if "running_var" in n_:
                b.copy_(torch.rand(b.shape, generator=g) + 0.5)
    return m


@pytest.mark.parametrize("cfg", [
    dict(P=20000, d=64, h=4, ff=128, blocks=1),                                     # BASELINE config 1 shape
    dict(P=20000, d=128, h=8, ff=256, blocks=2),
    dict(P=6000, d=128, h=8, ff=256, blocks=1, layer_cfg=dict(cosine=True, tau_min=0.01)),
    dict(P=6000, d=128, h=8, ff=256, blocks=1, layer_cfg=dict(cosine=True, non_shared_tau=True, post_norm=False)),
    dict(P=6000, d=64, h=8, ff=96, blocks=1, layer_cfg=dict(use_bn=True), act="relu", in_channel=64),
])
def test_sstv2_fp32_parity(cuda, cfg):
    """SSTv2 (sparse path) fp32: <= 1e-3 relative to the oracle (north_star tolerance), flat voxel order."""
    from sst_b200.sst_modules import SSTInputLayerV2
    d = cfg["d"]
    feats, coors = _voxels((1000,), cfg["P"], C=cfg.get("in_channel") or d)
    m = _sst_pair(d, cfg["h"], cfg["ff"], cfg["blocks"], cfg.get("layer_cfg"), cfg.get("act", "gelu"), cfg.get("in_channel"))
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    w = {k: v.clone() for k, v in m.state_dict().items()}
    lin0 = "linear0.weight" in w
    f_in = torch.nn.functional.linear(feats, w["linear0.weight"], w["linear0.bias"]) if lin0 else feats
    info_o = O.input_layer_v2(f_in, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    w_o = {k: v for k, v in w.items() if not k.startswith("linear0")}
    ref = O.sstv2_forward(info_o, w_o, [cfg["h"]] * cfg["blocks"], cfg["blocks"], cfg.get("act", "gelu"),
                          cfg.get("layer_cfg") or {})
    m = m.to(cuda)
    with torch.no_grad():
        info_g = il(feats.to(cuda), coors.to(cuda), 1)
        got = m(info_g)[0]["voxel_feats"].cpu()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-3, err
    torch.testing.assert_close(got, ref, rtol=1e-3, atol=2e-3)


@pytest.mark.parametrize("P,blocks", [(20000, 1), (150000, 6)])
def test_sstv2_bf16_parity(cuda, P, blocks):
    """bf16 tensor-core path (wgmma GEMMs, fp32 accumulate/softmax/LN): <= 1e-2 relative (north_star tolerance)."""
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels((1000,), P, C=128)
    m = _sst_pair(128, 8, 256, blocks)
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    w = {k: v.clone() for k, v in m.state_dict().items()}
    info_o = O.input_layer_v2(feats, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    ref = O.sstv2_forward(info_o, w, [8] * blocks, blocks)
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        info_g = il(feats.to(cuda), coors.to(cuda), 1)
        got = m(info_g)[0]["voxel_feats"].cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, err
    # element-wise as well: every output within 1e-2 relative, small outputs within 1e-2 of the output scale
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2 * ref.abs().max().item())
    # mean error is an order of magnitude below the bound (catches a systematically biased path that max-norm would pass)
    assert (got - ref).abs().mean().item() / ref.abs().mean().item() < 2e-3
    # and the fp32 path on the same inputs agrees with the oracle to fp32 accuracy
    m.precision = "fp32"
    with torch.no_grad():
        got32 = m(info_g)[0]["voxel_feats"].cpu()
    assert (got32 - ref).abs().max().item() / ref.abs().max().item() < 1e-3


@pytest.mark.parametrize("name,lc,P,blocks", [
    ("cosine, one tau per layer", dict(cosine=True, tau_min=0.01), 6000, 1),
    ("cosine, tau per head", dict(cosine=True, non_shared_tau=True, tau_min=0.01), 20000, 2),
    ("eval BatchNorm", dict(use_bn=True), 20000, 2),
    ("configs/fsd SST encoder: BatchNorm + cosine", dict(use_bn=True, cosine=True, tau_min=0.01), 150000, 4),
])
def test_sstv2_tensor_path_variants(cuda, name, lc, P, blocks):
    """precision='bf16' on the FUSED path (2 launches per layer) for the layer_cfg variants the reference's configs use with the
    SST-6 shape: cosine attention (sst_waymoD5_1x_3class_centerhead.py:75: 1/|q|, 1/|k| and 1/tau applied to the fp32 scores of the
    tensor-core kernel), eval-mode BatchNorm (folded scale / shift in the chain epilogues) and both together
    (configs/fsd/fsd_waymoD1_1x_sst_encoder.py:70).  Same <= 1e-2 bound as the plain path, max-norm and element-wise."""
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels((1000,), P, C=128)
    m = _sst_pair(128, 8, 256, blocks, lc)
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    w = {k: v.clone() for k, v in m.state_dict().items()}
    info_o = O.input_layer_v2(feats, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    ref = O.sstv2_forward(info_o, w, [8] * blocks, blocks, "gelu", lc)
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        got = m(il(feats.to(cuda), coors.to(cuda), 1))[0]["voxel_feats"].cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-2, (name, err)
    torch.testing.assert_close(got, ref, rtol=1e-2, atol=1e-2 * ref.abs().max().item())


def test_sstv2_tensor_path_variants_run_fused(cuda):
    """The variants above really take the fused stack path (2 kernels per layer): the frame graph of an engine built with cosine
    attention has exactly as many kernel nodes as the plain one, BatchNorm + cosine one more (the per-frame BatchNorm fold); the
    unfused fallback would add 3 launches per layer."""
    from sst_b200 import flagship as fl
    from sst_b200.engine import SSTEngine
    counts = {}
    for name, lc in (("plain", {}), ("cosine", dict(cosine=True, tau_min=0.01)), ("bn_cosine", dict(use_bn=True, cosine=True, tau_min=0.01))):
        cfg = fl.sst_cfg(num_blocks=2)
        cfg["backbone"]["layer_cfg"] = lc
        vfe, il, bb = fl.build_sst(cfg)
        eng = SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe.to(cuda), il, bb.to(cuda), max_points=20000, batch_size=1, precision="bf16", device=cuda)
        counts[name] = eng.launches_per_frame
    assert counts["cosine"] == counts["plain"], counts
    assert counts["bn_cosine"] == counts["plain"] + 1, counts


@pytest.mark.parametrize("layer_cfg,act,d,ff", [(dict(use_bn=True), "relu", 128, 256), (dict(post_norm=False), "gelu", 128, 256),
                                                ({}, "gelu", 64, 128)])
def test_sstv2_tensor_path_refuses_other_variants(cuda, layer_cfg, act, d, ff):
    """The tensor-core path is built for the reference's shipped shape (d_model 128, dim_ff 256, post-norm, gelu; LayerNorm or
    BatchNorm, plain or cosine attention).  Asking for it with relu / pre-norm / another width fails loudly - it never silently runs
    the fp32 kernels instead."""
    from sst_b200._lib import SSTB200Error
    from sst_b200.sst_modules import SSTInputLayerV2
    feats, coors = _voxels((1000,), 3000, C=d)
    m = _sst_pair(d, 8, ff, 1, layer_cfg, act).to(cuda)
    m.precision = "bf16"
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    with torch.no_grad(), pytest.raises(SSTB200Error, match="tensor-core path"):
        m(il(feats.to(cuda), coors.to(cuda), 1))


@pytest.mark.parametrize("B,C,ny,nx,M", [(2, 128, 468, 468, 40000), (1, 37, 50, 45, 700), (3, 64, 33, 32, 0), (1, 300, 40, 100, 1500)])
def test_recover_bev_exact(cuda, B, C, ny, nx, M):
    """SSTv2.recover_bev (sst_v2.py:161-196) is pure data movement: bit-exact against the oracle, including the zero fill."""
    from sst_b200.sst_modules import SSTv2
    g = torch.Generator().manual_seed(M + C)
    cells = torch.randperm(B * ny * nx, generator=g)[:M]
    b, rem = cells // (ny * nx), cells % (ny * nx)
    coors = torch.stack([b, torch.zeros_like(b), rem // nx, rem % nx], 1)
    feat = torch.randn(M, C, generator=g)
    m = SSTv2(d_model=[C], nhead=[1], num_blocks=0, dim_feedforward=[C], output_shape=[ny, nx], num_attached_conv=0, to_bev=True)
    got = m.recover_bev(feat.to(cuda), coors.to(cuda), B)
    assert torch.equal(got.cpu(), O.recover_bev(feat, coors, B, (ny, nx)))


def test_recover_bev_rejects_out_of_canvas(cuda):
    from sst_b200._lib import SSTB200Error
    from sst_b200.sst_modules import SSTv2
    m = SSTv2(d_model=[8], nhead=[1], num_blocks=0, dim_feedforward=[8], output_shape=[10, 10], num_attached_conv=0, to_bev=True)
    coors = torch.tensor([[0, 0, 3, 12]], device=cuda)
    with pytest.raises(SSTB200Error):
        m.recover_bev(torch.ones(1, 8, device=cuda), coors, 1)


def test_sstv2_to_bev_with_attached_convs(cuda):
    """Config 2 (ii): encoder stack -> BEV canvas -> the attached dense convs (cuDNN through torch; boundary layers, SURVEY 8f
    next-2).  The canvas feeding the convs must equal the oracle's sparse output scattered by the oracle."""
    from sst_b200.sst_modules import SSTInputLayerV2, SSTv2
    feats, coors = _voxels((1000,), 8000, C=64)
    torch.manual_seed(0)
    m = SSTv2(d_model=[64], nhead=[4], num_blocks=1, dim_feedforward=[128], output_shape=[468, 468], num_attached_conv=2,
              conv_in_channel=64, conv_out_channel=64, to_bev=True).eval()
    il = SSTInputLayerV2((DROP_TRAIN, DROP_TEST), (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True).eval()
    w = {k: v.clone() for k, v in m.state_dict().items()}
    info_o = O.input_layer_v2(feats, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    w_o = {k: v for k, v in w.items() if not k.startswith("conv_layer")}
    canvas = O.sstv2_forward(info_o, w_o, [4], 1, "gelu", {}, to_bev=True, output_shape=(468, 468))
    cpu_m = torch.nn.Sequential(*[cl for cl in m.conv_layer])
    with torch.no_grad():
        ref = cpu_m(canvas)
        m = m.to(cuda)
        got = m(il(feats.to(cuda), coors.to(cuda), 1))[0].cpu()
    assert got.shape == ref.shape == (1, 64, 468, 468)
    err = (got - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-3, err
