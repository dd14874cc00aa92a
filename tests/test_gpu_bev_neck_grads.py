"""GPU: the backward passes of SSTv2.recover_bev (csrc/bev.cu) and Voxel2PointScatterNeck (csrc/neck.cu) against autograd through the
CPU oracle (pinned to the reference by tests/test_oracle_bev_neck_grads_vs_reference.py), and the two model families trained through
them: the SST BEV configs (encoder stack -> canvas -> attached convs) and FSD's segmentor front (voxel encoder -> sparse U-Net -> neck)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import spconv_oracle as SO
from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
# configs/sst_refactor/sst_waymoD5_1x_3class_8heads_v2.py (and configs/sst/sst_waymoD5_1x_3class_8heads.py): the attached convs
CONV_KWARGS = [dict(kernel_size=3, dilation=1, padding=1, stride=1), dict(kernel_size=3, dilation=1, padding=1, stride=1),
               dict(kernel_size=3, dilation=2, padding=2, stride=1)]


def _rel(a, b):
    return (a.detach().cpu().float() - b.detach().float()).abs().max().item() / max(b.detach().abs().max().item(), 1e-30)


# ---- recover_bev ----------------------------------------------------------------------------------------------------------------------
def _bev_rows(B, ny, nx, M, dup, seed):
    g = torch.Generator().manual_seed(seed)
    if M is None:  # config 2: the voxels of a synthetic sweep on the 468 x 468 grid
        c = torch.unique(O.dynamic_voxelize(O.synth_frame(seed, 100000), VS, RNG), dim=0)
        return torch.nn.functional.pad(c, (1, 0), value=0).long()
    cells = torch.randperm(B * ny * nx, generator=g)[:M]
    if dup:
        cells = torch.cat([cells, cells[torch.randint(0, M, (dup,), generator=g)]])
        cells = cells[torch.randperm(cells.numel(), generator=g)]
    b, rem = cells // (ny * nx), cells % (ny * nx)
    return torch.stack([b, torch.zeros_like(b), rem // nx, rem % nx], 1)


@pytest.mark.parametrize("B,C,ny,nx,M,dup", [(1, 128, 468, 468, None, 0), (2, 37, 50, 45, 700, 0), (2, 37, 50, 45, 0, 0),
                                             (2, 40, 30, 30, 500, 150), (1, 300, 40, 100, 1500, 0)])
def test_recover_bev_backward_exact(cuda, B, C, ny, nx, M, dup):
    """d voxel_feat[m] = d canvas[b_m, :, y_m, x_m], bit-exact against the oracle's autograd (index_put backward), duplicated cells
    included; the forward under autograd is the no-grad forward."""
    from sst_b200.sst_modules import SSTv2
    coors = _bev_rows(B, ny, nx, M, dup, seed=11 + C)
    if M is None:
        assert 20000 < coors.shape[0] < 40000
    g = torch.Generator().manual_seed(C)
    feat = torch.randn(coors.shape[0], C, generator=g)
    probe = torch.randn(B, C, ny, nx, generator=g)
    xo = feat.clone().requires_grad_(True)
    (O.recover_bev(xo, coors, B, (ny, nx)) * probe).sum().backward()
    m = SSTv2(d_model=[C], nhead=[1], num_blocks=0, dim_feedforward=[C], output_shape=[ny, nx], num_attached_conv=0, to_bev=True)
    x = feat.to(cuda).requires_grad_(True)
    canvas = m.recover_bev(x, coors.to(cuda), B)
    assert canvas.requires_grad
    if not dup:
        with torch.no_grad():
            assert torch.equal(canvas.detach(), m.recover_bev(feat.to(cuda), coors.to(cuda), B))
    canvas.backward(probe.to(cuda))
    assert torch.equal(x.grad.cpu(), xo.grad)


# ---- Voxel2PointScatterNeck ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,M,C,with_xyz,norm", [(150000, 30000, 128, True, False), (5000, 700, 16, True, True), (5000, 700, 37, False, False),
                                                (33, 5, 3, True, False)])
def test_voxel2point_neck_backward(cuda, N, M, C, with_xyz, norm):
    """grad_voxel_feats within 1e-6 of max|ref| of float64 autograd; a voxel with one kept point bit-exact; padded and unreferenced voxels
    exactly 0; two backward passes give the same bits."""
    from sst_b200.neck_modules import Voxel2PointScatterNeck
    g = torch.Generator().manual_seed(N + C)
    pts = O.synth_frame(3, N, extra_dims=1)
    coors = torch.nn.functional.pad(O.dynamic_voxelize(pts, VS, RNG), (1, 0), value=0).long()
    vf = torch.randn(M, C, generator=g)
    vf[::7] = -1.0
    inds = torch.randint(0, M, (N,), generator=g)
    xo = vf.double().requires_grad_(True)
    o_out, o_mask = O.voxel2point_neck(pts.double(), coors, xo, inds, VS, RNG, with_xyz, norm)
    probe = torch.randn(o_out.shape, generator=g)
    (o_out * probe.double()).sum().backward()
    ref = xo.grad
    neck = Voxel2PointScatterNeck(point_cloud_range=RNG, voxel_size=VS, with_xyz=with_xyz, normalize_local_xyz=norm).train()
    grads = []
    for _ in range(2):
        x = vf.to(cuda).requires_grad_(True)
        out, mask = neck(pts.to(cuda), coors.to(cuda), x, inds.to(cuda))
        assert torch.equal(mask.cpu(), o_mask) and not mask.requires_grad
        with torch.no_grad():
            out_ng, _ = neck(pts.to(cuda), coors.to(cuda), vf.to(cuda), inds.to(cuda))
        assert torch.equal(out.detach(), out_ng)
        out.backward(probe.to(cuda))
        grads.append(x.grad.cpu())
    got = grads[0]
    assert torch.equal(grads[0], grads[1])
    assert (got.double() - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()
    cnt = torch.bincount(inds[o_mask], minlength=M)
    if N >= 5000:  # single-point voxels, and (at 150k points) voxels no point references beside the padded ones
        assert int((cnt == 1).sum()) > 0
        assert N < 150000 or int(((cnt == 0) & (torch.arange(M) % 7 != 0)).sum()) > 0
    assert torch.equal(got[cnt == 1], ref[cnt == 1].float())
    assert int((got[cnt == 0] != 0).sum()) == 0
    assert int((got[::7] != 0).sum()) == 0


def test_voxel2point_neck_refuses_point_gradients(cuda):
    from sst_b200.neck_modules import Voxel2PointScatterNeck
    neck = Voxel2PointScatterNeck(point_cloud_range=RNG, voxel_size=VS)
    pts = torch.zeros(4, 3, device=cuda, requires_grad=True)
    with pytest.raises(NotImplementedError):
        neck(pts, torch.zeros(4, 4, dtype=torch.long, device=cuda), torch.zeros(2, 8, device=cuda, requires_grad=True),
             torch.tensor([0, 1, 1, 0], device=cuda))


# ---- SST BEV configs: encoder stack -> canvas -> attached convs ----------------------------------------------------------------------
def _bev_voxels(B, side, per_sample, seed):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b in range(B):
        cells = torch.randperm(side * side, generator=g)[:per_sample]
        rows.append(torch.stack([torch.full_like(cells, b), torch.zeros_like(cells), cells // side, cells % side], 1))
    coors = torch.cat(rows)
    return torch.randn(coors.shape[0], 128, generator=g), coors


def _randomize_stack(bb, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n_, q in bb.named_parameters():
            if q.dim() == 1 and n_.startswith("block_list"):
                q.copy_(torch.randn(q.shape, generator=g) * 0.1 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))


def _oracle_convs(x, w, eps=1e-3):
    """The attached convs of SSTv2.forward (sst_v2.py:135-146): Conv2d (no bias) -> training-mode naiveSyncBN2d (one process: batch
    statistics) -> ReLU."""
    for i, kw in enumerate(CONV_KWARGS):
        x = F.conv2d(x, w[f"conv_layer.{i}.0.weight"], None, stride=kw["stride"], padding=kw["padding"], dilation=kw["dilation"])
        x = F.batch_norm(x, None, None, w[f"conv_layer.{i}.1.weight"], w[f"conv_layer.{i}.1.bias"], True, 0.0, eps)
        x = F.relu(x)
    return x


@pytest.mark.parametrize("version", ["v2", "v1"])
def test_sst_bev_config_gradients(cuda, version):
    """bf16 SSTv2 (configs/sst_refactor) or SSTv1 with SSTInputLayer (configs/sst) in training mode, 2 blocks, to_bev with the three
    attached convs (training-mode BN), on a cropped 96 x 96 canvas.  The ReLUs of the dense head switch wherever the bf16 forward and the
    fp32 oracle disagree in sign, and each switch moves one gradient element by its full size, so the check is split at the canvas: the dense head's gradients against fp32 autograd over the canvas this run produced, and the canvas
    gradient this run produced sent back through the oracle's encoder stack.  Every parameter and the input gradient within the
    bf16 tolerance of test_gpu_train (2e-2 of max-abs), and every encoder layer receives a gradient."""
    from sst_b200.sst_modules import SSTInputLayer, SSTInputLayerV2, SSTv1, SSTv2
    side, B = 96, 2
    feats, coors = _bev_voxels(B, side, 2500, seed=21)
    common = dict(d_model=[128] * 2, nhead=[8] * 2, num_blocks=2, dim_feedforward=[256] * 2, output_shape=[side, side], num_attached_conv=3,
                  conv_kwargs=CONV_KWARGS, conv_in_channel=128, conv_out_channel=128, precision="bf16")
    torch.manual_seed(5)
    if version == "v2":
        bb = SSTv2(to_bev=True, **common)
        il = SSTInputLayerV2(DROP_TEST, (12, 12, 1), (side, side, 1), shuffle_voxels=False, mute=True)
    else:
        bb = SSTv1(drop_info=DROP_TEST, window_shape=(12, 12), pos_temperature=10000, normalize_pos=False, **common)
        il = SSTInputLayer(drop_info=DROP_TEST, shifts_list=[(0, 0), (6, 6)], window_shape=(12, 12),
                           point_cloud_range=[0, 0, -2, side, side, 4], voxel_size=(1.0, 1.0, 6), shuffle_voxels=False)
    _randomize_stack(bb, 6)
    w = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in bb.state_dict().items()}
    probe = torch.randn(B, 128, side, side, generator=torch.Generator().manual_seed(7))
    # CUDA, keeping the canvas and its gradient
    seen = {}
    recover_bev = bb.recover_bev

    def keep_canvas(*args):
        seen["canvas"] = recover_bev(*args)
        seen["canvas"].retain_grad()
        return seen["canvas"]

    bb.recover_bev = keep_canvas
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        bb = bb.to(cuda).train()
        x = feats.to(cuda).requires_grad_(True)
        y = bb(il.train()(x, coors.to(cuda), B))[0]  # v1: the input layer's tuple, v2: its voxel_info dict
        (y * probe.to(cuda)).sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    canvas, d_canvas = seen["canvas"].detach().cpu(), seen["canvas"].grad.cpu()
    # oracle, dense head over this run's canvas (fp32 CPU autograd)
    co = canvas.clone().requires_grad_(True)
    yo = _oracle_convs(co, w)
    (yo * probe).sum().backward()
    assert _rel(y, yo) < 1e-4 and _rel(d_canvas, co.grad) < 1e-4
    # oracle, encoder stack and canvas, fed this run's canvas gradient
    xo = feats.clone().requires_grad_(True)
    info_o = O.input_layer_v2(xo, coors, DROP_TEST, (12, 12, 1), (side, side, 1))
    canvas_o = O.sstv2_forward(info_o, w, [8, 8], 2, to_bev=True, output_shape=(side, side))
    assert _rel(canvas, canvas_o) < 2e-2
    canvas_o.backward(d_canvas)
    assert _rel(x.grad, xo.grad) < 2e-2, f"d input: {_rel(x.grad, xo.grad)}"
    bad, n_enc = {}, 0
    for name, p in bb.named_parameters():
        assert p.grad is not None, name
        if name.startswith("block_list"):
            assert p.grad.abs().max().item() > 0, f"{name} received no gradient"
            n_enc += 1
        r = _rel(p.grad, w[name].grad)
        if r > (2e-2 if name.startswith("block_list") else 1e-4):
            bad[name] = r
    assert n_enc == 2 * 2 * 12 and not bad, f"parameter gradients off (bf16 tolerance 2e-2 of max-abs; dense head 1e-4): {bad}"


# ---- FSD segmentor front: voxel encoder -> sparse U-Net -> neck ---------------------------------------------------------------------
def test_fsd_segmentor_front_gradients(cuda):
    """VoteSegmentor.extract_feat (single_stage_fsd.py:228-250) trained through this library: DynamicScatterVFE (training-mode BN) ->
    SimpleSparseUNet (SO.SP_UNET, frozen BN statistics as in test_unet_gradients) -> Voxel2PointScatterNeck(with_xyz) -> probe loss;
    every parameter gradient against autograd through the oracle chain."""
    from sst_b200 import registry
    cfg = dict(SO.SP_UNET)
    vs, rng = (0.5, 0.5, 0.5), [-8, -8, -2, 8, 8, 2.5]  # grid 32 x 32 x 9 = SP_UNET's sparse shape
    norm = dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01)
    torch.manual_seed(3)
    vfe = registry.MODELS.build(dict(type='DynamicScatterVFE', in_channels=5, feat_channels=[16, cfg["in_channels"]], with_cluster_center=True,
                                     with_voxel_center=True, voxel_size=vs, point_cloud_range=rng, norm_cfg=norm, unique_once=True)).train()
    net = registry.MODELS.build(dict(type="SimpleSparseUNet", **cfg)).eval()
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.2)
    neck = registry.MODELS.build(dict(type='Voxel2PointScatterNeck', voxel_size=vs, point_cloud_range=rng, with_xyz=True))
    P = 3000
    pts = torch.cat([torch.cat([O.synth_frame(30 + b, P) * torch.tensor([0.1, 0.1, 0.7]), torch.rand(P, 2, generator=g)], 1) for b in range(2)])
    co = torch.cat([F.pad(O.dynamic_voxelize(pts[b * P:(b + 1) * P], vs, rng), (1, 0), value=b) for b in range(2)]).long()
    # oracle
    wv = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in vfe.state_dict().items()}
    wu = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in net.state_dict().items()}
    of, oc, oinv = O.dynamic_scatter_vfe_forward(pts, co, wv, vs, rng, 2, training=True)
    uf, _ = SO.sparse_unet_forward(wu, of, oc.int(), 2, cfg["sparse_shape"], cfg["encoder_channels"], cfg["encoder_paddings"],
                                   cfg["decoder_channels"], cfg["decoder_paddings"])
    out_o, mask_o = O.voxel2point_neck(pts, co, uf, oinv, vs, rng)
    probe = torch.randn(out_o.shape, generator=torch.Generator().manual_seed(9))
    (out_o * probe).sum().backward()
    # CUDA
    vfe, net = vfe.to(cuda), net.to(cuda)
    vf, vc, inv = vfe(pts.to(cuda), co.to(cuda), return_inv=True)
    x = net(dict(voxel_feats=vf, voxel_coors=vc))[0]
    out, mask = neck(pts.to(cuda), co.to(cuda), x["voxel_feats"], inv)
    assert torch.equal(mask.cpu(), mask_o) and _rel(out, out_o) < 1e-3
    (out * probe.to(cuda)).sum().backward()
    bad, n = {}, 0
    for mod, w in ((vfe, wv), (net, wu)):
        for name, p in mod.named_parameters():
            assert p.grad is not None and p.grad.abs().max().item() > 0, name
            r = _rel(p.grad, w[name].grad)
            if r > 2e-3:
                bad[name] = r
            n += 1
    assert n > 60 and not bad, bad


# ---- the regression: a BEV training loop reaches the encoder and the voxel encoder ----------------------------------------------------
def test_bev_training_loop_reaches_the_encoder(cuda):
    """Ten FlatAdamW steps on DynamicVFE + SSTv2(to_bev=True, 3 attached convs) with a stand-in loss on the canvas: the loss decreases and,
    at every step, every voxel-encoder and encoder-layer parameter receives a non-zero gradient (the gradient, not the parameter change:
    weight decay alone moves every parameter)."""
    from sst_b200 import flagship as fl
    from sst_b200.train import FlatAdamW
    cfg = fl.sst_cfg(num_blocks=2)
    cfg["backbone"].update(precision="bf16", to_bev=True, num_attached_conv=3, conv_kwargs=CONV_KWARGS, conv_in_channel=128,
                           conv_out_channel=128)
    vfe, il, bb = fl.build_sst(cfg, seed=4)
    vfe, bb = vfe.to(cuda).train(), bb.to(cuda).train()
    il.train()
    pts = torch.cat([O.synth_frame(51, 15000), O.synth_frame(52, 12000)])
    c3 = O.dynamic_voxelize(pts, VS, RNG)
    coors = torch.cat([F.pad(c3[:15000], (1, 0), value=0), F.pad(c3[15000:], (1, 0), value=1)]).to(cuda)
    pts = pts.to(cuda)
    opt = FlatAdamW(list(vfe.parameters()) + list(bb.parameters()), lr=2e-3, weight_decay=0.05)
    watched = [(n, p) for n, p in vfe.named_parameters()] + [(n, p) for n, p in bb.named_parameters() if n.startswith("block_list")]
    assert len(watched) > 48
    losses = []
    for step in range(10):
        opt.zero_grad()
        vf, vc = vfe(pts, coors)
        canvas = bb(il(vf, vc, 2))[0]
        loss = canvas.square().mean()
        loss.backward()
        dead = [n for n, p in watched if not p.grad.abs().max().item() > 0]
        assert not dead, f"step {step}: no gradient reached {dead}"
        losses.append(loss.item())
        opt.step()
    assert losses[-1] < losses[0], losses
