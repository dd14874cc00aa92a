"""GPU parity of the whole config-2 style path (voxelize -> DynamicVFE -> SSTInputLayerV2 -> SSTv2) through the
registered modules and through the sync-free engine (CUDA graph), against the CPU oracle."""
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu


def _oracle_path(pts_list, vfe, bb, cfg, fl):
    coors = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(p, fl.VOXEL_SIZE, fl.PC_RANGE), (1, 0), value=b)
                       for b, p in enumerate(pts_list)])
    pts = torch.cat(pts_list)
    wv = {k: v.cpu() for k, v in vfe.state_dict().items()}
    vf, vc = O.dynamic_vfe_forward(pts, coors, wv, fl.VOXEL_SIZE, fl.PC_RANGE, 2)
    info = O.input_layer_v2(vf, vc, fl.DROP_TEST, fl.WINDOW_SHAPE, (468, 468, 1))
    wb = {k: v.cpu() for k, v in bb.state_dict().items()}
    nb = cfg['backbone']['num_blocks']
    out = O.sstv2_forward(info, wb, cfg['backbone']['nhead'], nb)
    return vf, vc, out


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("P,batch,extra", [(20000, 1, 0), (8000, 3, 2), (150000, 1, 0)])
def test_vfe_matches_oracle(cuda, P, batch, extra, precision):
    from sst_b200 import flagship as fl, ops
    cfg = fl.sst_cfg(num_blocks=1, in_channels=3 + extra)
    vfe, il, bb = fl.build_sst(cfg)
    pts_list = [O.synth_frame(40 + b, P, extra_dims=extra) for b in range(batch)]
    vf_o, vc_o, _ = _oracle_path(pts_list, vfe, bb, cfg, fl)
    vfe = vfe.to(cuda)
    vox = ops.Voxelization(fl.VOXEL_SIZE, fl.PC_RANGE, -1, (-1, -1))
    coors = torch.cat([torch.nn.functional.pad(vox(p.to(cuda)), (1, 0), value=b) for b, p in enumerate(pts_list)])
    vfe.precision = precision
    vf, vc = vfe(torch.cat(pts_list).to(cuda), coors)
    assert torch.equal(vc.cpu(), vc_o)
    if precision == "fp32":
        torch.testing.assert_close(vf.cpu(), vf_o, rtol=1e-4, atol=1e-4)
    else:  # second VFE layer with bf16 operands on the tensor cores: north_star bf16 tolerance
        assert (vf.cpu() - vf_o).abs().max().item() / vf_o.abs().max().item() < 1e-2


def test_dynamic_scatter_vfe_matches_oracle(cuda):
    from sst_b200.voxel_modules import DynamicScatterVFE
    vs, rng = (0.25, 0.25, 0.2), [-80, -80, -2, 80, 80, 4]
    torch.manual_seed(0)
    m = DynamicScatterVFE(in_channels=5, feat_channels=[64, 64], with_cluster_center=True, with_voxel_center=True,
                          voxel_size=vs, point_cloud_range=rng, norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01),
                          unique_once=True, rel_dist_scaler=10.0).eval()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.normal_(0, 0.5)
            mod.running_var.uniform_(0.5, 2)
    pts = torch.cat([torch.cat([O.synth_frame(3 + b, 15000), torch.rand(15000, 2)], 1) for b in range(2)])
    co = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(pts[b * 15000:(b + 1) * 15000], vs, rng), (1, 0), value=b)
                    for b in range(2)]).long()
    ref = O.dynamic_scatter_vfe_forward(pts, co, dict(m.state_dict()), vs, rng, 2, rel_dist_scaler=10.0)
    m = m.to(cuda)
    got = m(pts.to(cuda), co.to(cuda), return_inv=True)
    assert torch.equal(got[1].cpu(), ref[1]) and torch.equal(got[2].cpu(), ref[2])
    torch.testing.assert_close(got[0].cpu(), ref[0], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-3), ("bf16", 1e-2)])
def test_engine_matches_oracle(cuda, precision, tol):
    """Sync-free engine (CUDA graph, capacity-sized buffers, padded tail rows) == oracle, batch of 2 frames."""
    from sst_b200 import flagship as fl
    from sst_b200.engine import SSTEngine
    cfg = fl.sst_cfg(num_blocks=2)
    vfe, il, bb = fl.build_sst(cfg)
    pts_list = [O.synth_frame(70 + b, 12000) for b in range(2)]
    vf_o, vc_o, out_o = _oracle_path(pts_list, vfe, bb, cfg, fl)
    eng = SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe.to(cuda), il, bb.to(cuda), max_points=30000, batch_size=2,
                    precision=precision, device=cuda)
    pts = torch.cat(pts_list).to(cuda)
    offs = torch.tensor([0, 12000, 24000], dtype=torch.int32, device=cuda)
    for _ in range(2):  # replay twice: the graph must be re-entrant
        eng.load_frames_device(pts, offs)
        feats, coors, num = eng.run()
        torch.cuda.synchronize()
    M = int(num.item())
    assert M == vc_o.shape[0]
    assert torch.equal(coors[:M].cpu(), vc_o)
    got = feats[:M].cpu()
    err = (got - out_o).abs().max().item() / out_o.abs().max().item()
    assert err < tol, err


def test_engine_host_api_with_predicted_row_count(cuda):
    """forward_host / submit_host + collect_host on pinned HOST buffers: the D2H of the result is enqueued for a predicted row
    count; frames with fewer, equal and MORE voxels than predicted all return exactly the rows the device path returns."""
    from sst_b200 import flagship as fl
    from sst_b200.engine import SSTEngine
    cfg = fl.sst_cfg(num_blocks=1)
    vfe, il, bb = fl.build_sst(cfg)
    eng = SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe.to(cuda), il, bb.to(cuda), max_points=30000, batch_size=1, precision="bf16", device=cuda)
    out_f = torch.empty((30000, eng.d), dtype=torch.float32).pin_memory()
    out_c = torch.empty((30000, 4), dtype=torch.int32).pin_memory()
    seen = []
    for seed, P in [(1, 8000), (2, 8000), (3, 5000), (4, 30000), (5, 9000)]:   # 4th frame: far more voxels than predicted
        pts = O.synth_frame(seed, P)
        offs = torch.tensor([0, P], dtype=torch.int32)
        eng.load_frames_device(pts.to(cuda), offs.to(cuda))
        feats, coors, num = eng.run()
        torch.cuda.synchronize()
        M_ref = int(num.item())
        ref_f, ref_c = feats[:M_ref].cpu(), coors[:M_ref].cpu()
        out_f.fill_(float("nan"))
        M = eng.forward_host(pts.pin_memory(), offs.pin_memory(), out_f, out_c)
        eng.stream.synchronize()
        assert M == M_ref
        assert torch.equal(out_f[:M], ref_f) and torch.equal(out_c[:M], ref_c)
        assert eng.d2h_rows >= M
        seen.append((M, eng.d2h_rows))
    assert seen[0][1] == seen[0][0]            # no prediction for the first frame: exactly M rows
    assert seen[1][1] > seen[1][0]             # predicted: a little more than needed
    assert seen[3][0] > seen[2][1]             # the big frame really exceeded the prediction


@pytest.mark.parametrize("mode", ["max", "avg"])
def test_dynamic_scatter_vfe_wide_input(cuda, mode):
    """FSDv2's virtual-voxel encoder shape (configs/fsdv2: in_channels 67 -> [64, 128], SURVEY config 5): beyond the fused
    kernels' 16 decorated dims, served by the row-GEMM path; coordinates / inverse bit-exact, features <= 1e-3."""
    from sst_b200.voxel_modules import DynamicScatterVFE
    vs, rng = (0.4, 0.4, 0.4), [-51.2, -51.2, -5, 51.2, 51.2, 3]
    torch.manual_seed(0)
    m = DynamicScatterVFE(in_channels=67, feat_channels=[64, 128], with_cluster_center=True, with_voxel_center=True, voxel_size=vs,
                          point_cloud_range=rng, norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01), unique_once=True,
                          rel_dist_scaler=10.0, mode=mode).eval()
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm1d):
            mod.running_mean.normal_(0, 0.5)
            mod.running_var.uniform_(0.5, 2)
    n = 9000
    pts = torch.cat([torch.cat([O.synth_frame(30 + b, n) * 0.6, torch.randn(n, 64)], 1) for b in range(2)])
    co = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(pts[b * n:(b + 1) * n], vs, rng), (1, 0), value=b) for b in range(2)]).long()
    ref = O.dynamic_scatter_vfe_forward(pts, co, dict(m.state_dict()), vs, rng, 2, rel_dist_scaler=10.0, mode=mode)
    m = m.to(cuda)
    got = m(pts.to(cuda), co.to(cuda), return_inv=True)
    assert torch.equal(got[1].cpu(), ref[1]) and torch.equal(got[2].cpu(), ref[2])
    err = (got[0].cpu() - ref[0]).abs().max().item() / ref[0].abs().max().item()
    assert err < 1e-3, err


def test_fsd_segmentation_front_pipeline(cuda):
    """VoteSegmentor.extract_feat (mmdet3d/models/detectors/single_stage_fsd.py:227-249) through the registered modules with the configs/fsd
    type names - DynamicScatterVFE -> PseudoMiddleEncoderForSpconvFSD -> SimpleSparseUNet -> Voxel2PointScatterNeck - then the grouping
    stage (ClusterAssigner) on the per-point output: every hand-over matches the oracle chain (coordinates / masks / cluster ids exact)."""
    from oracle import fsd_oracle as FO, spconv_oracle as SO
    from sst_b200 import ops, registry
    vs, rng = (0.5, 0.5, 0.375), [-40, -40, -2, 40, 40, 4]         # grid 160 x 160 x 16
    norm = dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01)
    unet_cfg = dict(in_channels=32, sparse_shape=[16, 160, 160], norm_cfg=norm, base_channels=16, output_channels=16,
                    encoder_channels=((16,), (16, 16, 16), (32, 32, 32)), encoder_paddings=((1,), (1, 1, 1), (1, 1, 1)),
                    decoder_channels=((32, 32, 16), (16, 16, 16), (16, 16, 16)), decoder_paddings=((1, 1), (1, 0), (0, 1)))
    torch.manual_seed(1)
    vfe = registry.MODELS.build(dict(type='DynamicScatterVFE', in_channels=5, feat_channels=[32, 32], with_cluster_center=True,
                                     with_voxel_center=True, voxel_size=vs, point_cloud_range=rng, norm_cfg=norm, unique_once=True)).eval()
    me = registry.MODELS.build(dict(type='PseudoMiddleEncoderForSpconvFSD'))
    bb = registry.MODELS.build(dict(type='SimpleSparseUNet', **unet_cfg)).eval()
    neck = registry.MODELS.build(dict(type='Voxel2PointScatterNeck', voxel_size=vs, point_cloud_range=rng))
    g = torch.Generator().manual_seed(3)
    for m in list(vfe.modules()) + list(bb.modules()):
        if isinstance(m, torch.nn.BatchNorm1d):
            m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.2)
            m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
    P = 6000
    pts = torch.cat([torch.cat([O.synth_frame(7 + b, P) * torch.tensor([0.5, 0.5, 1.0]), torch.rand(P, 2, generator=g)], 1) for b in range(2)])
    co = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(pts[b * P:(b + 1) * P], vs, rng), (1, 0), value=b) for b in range(2)]).long()
    # oracle chain (CPU)
    vf_r, vc_r, inv_r = O.dynamic_scatter_vfe_forward(pts, co, dict(vfe.state_dict()), vs, rng, 2)
    uf_r, uc_r = SO.sparse_unet_forward(bb.state_dict(), vf_r, vc_r.int(), 2, unet_cfg["sparse_shape"], unet_cfg["encoder_channels"],
                                        unet_cfg["encoder_paddings"], unet_cfg["decoder_channels"], unet_cfg["decoder_paddings"])
    out_r, mask_r = O.voxel2point_neck(pts, co, uf_r, inv_r, vs, rng)
    # product chain (GPU)
    vfe, bb = vfe.to(cuda), bb.to(cuda)
    with torch.no_grad():
        vf, vc, inv = vfe(pts.to(cuda), co.to(cuda), return_inv=True)
        x = bb(me(vf, vc))[0]
        out, mask = neck(pts.to(cuda), co.to(cuda), x['voxel_feats'], inv, -1)
    assert torch.equal(vc.cpu(), vc_r) and torch.equal(inv.cpu(), inv_r)
    assert torch.equal(x['voxel_coors'].cpu().long(), vc_r) and x['batch_size'] == 2
    torch.testing.assert_close(x['voxel_feats'].cpu(), uf_r, rtol=1e-3, atol=1e-4)
    assert torch.equal(mask.cpu(), mask_r)
    torch.testing.assert_close(out.cpu(), out_r, rtol=1e-3, atol=1e-4)
    # grouping on the points that survived (their xyz stand in for the voted centres; lattice coordinates keep the voxel means exact)
    from sst_b200.fsd_modules import ClusterAssigner
    ca = ClusterAssigner(cluster_voxel_size=dict(Car=(0.3, 0.3, 6)), min_points=2, point_cloud_range=rng, connected_dist=dict(Car=0.6),
                         class_names=['Car']).train()
    centres = torch.round(pts[mask_r][:, :3] * 64) / 64
    bidx = co[mask_r][:, 0].int()
    inds, valid = ca([centres.to(cuda)], [bidx.to(cuda)])
    ref_inds, ref_valid = FO.cluster_assigner_single_class(centres, bidx, (0.3, 0.3, 6), 2, rng, 0.6)
    assert torch.equal(valid[0].cpu(), ref_valid)
    assert torch.equal(inds[0][:, 1:].cpu().int(), ref_inds) and int(inds[0][:, 0].abs().sum()) == 0


def test_dynamic_scatter_vfe_training_gradients(cuda):
    """DynamicScatterVFE.train(): the composition over ops.unique_rows / ops.segment_reduce (forward + backward kernels) and torch Linear /
    naiveSyncBN matches the oracle's training=True restatement (pinned to the reference class in train mode): outputs, the input gradient
    and every parameter gradient; then the FSD trainable chain DynamicScatterVFE -> SimpleSparseUNet takes one optimiser step"""
    from sst_b200 import registry
    vs, rng = (0.25, 0.25, 0.2), [-80, -80, -2, 80, 80, 4]
    norm = dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01)
    torch.manual_seed(0)
    m = registry.MODELS.build(dict(type='DynamicScatterVFE', in_channels=5, feat_channels=[32, 32], with_cluster_center=True, with_voxel_center=True,
                                   voxel_size=vs, point_cloud_range=rng, norm_cfg=norm, unique_once=True, rel_dist_scaler=10.0)).train()
    pts = torch.cat([torch.cat([O.synth_frame(3 + b, 3000), torch.rand(3000, 2)], 1) for b in range(2)])
    co = torch.cat([torch.nn.functional.pad(O.dynamic_voxelize(pts[b * 3000:(b + 1) * 3000], vs, rng), (1, 0), value=b) for b in range(2)]).long()
    w = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in m.state_dict().items()}
    x_ref = pts.clone().requires_grad_(True)
    of, oc, oinv = O.dynamic_scatter_vfe_forward(x_ref, co, w, vs, rng, 2, rel_dist_scaler=10.0, training=True)
    probe = torch.randn(of.shape, generator=torch.Generator().manual_seed(1))
    (of * probe).sum().backward()
    m = m.to(cuda)
    x = pts.to(cuda).requires_grad_(True)
    vf, vc, inv = m(x, co.to(cuda), return_inv=True)
    assert torch.equal(vc.cpu(), oc) and torch.equal(inv.cpu(), oinv)
    torch.testing.assert_close(vf.detach().cpu(), of.detach(), rtol=1e-4, atol=1e-4)
    (vf * probe.to(cuda)).sum().backward()
    torch.testing.assert_close(x.grad.cpu(), x_ref.grad, rtol=1e-3, atol=1e-4 * float(x_ref.grad.abs().max()))
    for name, p in m.named_parameters():
        torch.testing.assert_close(p.grad.cpu(), w[name].grad, rtol=1e-3, atol=2e-4 * float(w[name].grad.abs().max()) + 1e-7)
    # one training step of the FSD segmentation chain (voxel encoder -> sparse U-Net), every parameter receives a finite gradient
    unet = registry.MODELS.build(dict(type='SimpleSparseUNet', in_channels=32, sparse_shape=[32, 640, 640], norm_cfg=norm, base_channels=16,
                                      output_channels=16, encoder_channels=((16,), (16, 16), (32, 32)), encoder_paddings=((1,), (1, 1), (1, 1)),
                                      decoder_channels=((32, 32, 16), (16, 16, 16), (16, 16, 16)),
                                      decoder_paddings=((1, 1), (1, 0), (0, 1)))).to(cuda).train()
    params = list(m.parameters()) + list(unet.parameters())
    opt = torch.optim.AdamW(params, lr=1e-3)
    opt.zero_grad()
    vf, vc, inv = m(pts.to(cuda), co.to(cuda), return_inv=True)
    out = unet(dict(voxel_feats=vf, voxel_coors=vc))[0]["voxel_feats"]
    loss = out.float().square().mean()
    loss.backward()
    assert all(p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in params)
    assert sum(float(p.grad.abs().sum()) for p in unet.parameters()) > 0 and float(m.vfe_layers[0].linear.weight.grad.abs().sum()) > 0
    opt.step()
