"""GPU: sparse 3-D convolution (SURVEY 8f next-1) through the C ABI against
  * fixtures produced by the reference's own vendored spconv v1 layers / SimpleSparseUNet / VirtualVoxelMixer (tests/golden/spconv_*.npz),
  * the oracle's dense restatement (oracle/spconv_oracle.py, pinned to that reference in tests/test_oracle_spconv_vs_reference.py),
  * the reference's own CUDA spconv kernels on the same device tensors (oracle/_ref/sparse_conv_ext_ref*.so), at the FSD size,
  * size-independent properties at the FSD size (identity kernel, table transposition, fp32 path == tensor-core path).
Index work (output coordinates, neighbour tables) is bit-exact; features: fp32 path 1e-4, tensor-core path 1e-2 of max|ref|."""
import os

import numpy as np
import pytest
import torch

from oracle import spconv_oracle as SO

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def _sorted(f, c):
    c = c.long()
    order = torch.argsort(((c[:, 0] * 4096 + c[:, 1]) * 4096 + c[:, 2]) * 4096 + c[:, 3])
    return f[order], c[order].int()


def _close(a, ref, tol):
    a, ref = a.float().cpu(), ref.float().cpu()
    scale = ref.abs().max().item()
    err = (a - ref).abs().max().item() / max(scale, 1e-30)
    assert err < tol, f"max-norm error {err:.3e} >= {tol}"
    torch.testing.assert_close(a, ref, rtol=tol, atol=tol * scale)


@pytest.mark.parametrize("ks,stride,padding", [((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1)),
                                               ((3, 1, 1), (2, 1, 1), (0, 0, 0)), ((2, 2, 2), (2, 2, 2), (0, 0, 0)),
                                               ((3, 3, 3), (1, 1, 1), (1, 1, 1))])
def test_tables_bitexact(cuda, ks, stride, padding):
    from sst_b200 import spconv_modules as SP
    shape = [9, 40, 44]
    feats, coors = SO.synth_sparse(31, 3, shape, 1500, 4)
    oshape = SO.conv_output_size(shape, ks, stride, padding)
    oc_ref = SO.out_coors(coors, 3, shape, ks, stride, padding)
    oc = SP.conv_out_coors(coors.to(cuda), 3, shape, oshape, ks, stride, padding)
    assert torch.equal(oc.cpu(), oc_ref)
    nbr, inv = SP.conv_table(coors.to(cuda), oc, 3, shape, oshape, ks, stride, padding, want_nbr=True, want_inv=True)
    nbr_ref = SO.neighbour_table(coors, oc_ref, 3, shape, ks, stride, padding)
    assert torch.equal(nbr.cpu(), nbr_ref)
    # the transposed table holds exactly the same pairs
    kv = nbr_ref.shape[1]
    inv_ref = torch.full((coors.shape[0], kv), -1, dtype=torch.int32)
    o_idx, k_idx = torch.nonzero(nbr_ref >= 0, as_tuple=True)
    inv_ref[nbr_ref[o_idx, k_idx].long(), k_idx] = o_idx.int()
    assert torch.equal(inv.cpu(), inv_ref)


def test_subm_table_and_empty(cuda):
    from sst_b200 import spconv_modules as SP
    shape = [5, 30, 30]
    feats, coors = SO.synth_sparse(5, 2, shape, 700, 4)
    nbr, _ = SP.conv_table(coors.to(cuda), coors.to(cuda), 2, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
    assert torch.equal(nbr.cpu(), SO.neighbour_table(coors, coors, 2, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1]))
    assert torch.equal(nbr[:, 13].cpu(), torch.arange(coors.shape[0], dtype=torch.int32))   # centre offset = the row itself
    empty = torch.zeros((0, 4), dtype=torch.int32, device=cuda)
    assert SP.conv_out_coors(empty, 2, shape, [3, 15, 15], [3, 3, 3], [2, 2, 2], [1, 1, 1]).shape == (0, 4)
    with pytest.raises(Exception):   # a coordinate outside the grid is an error, not a silent drop
        bad = coors.clone()
        bad[3, 2] = 30
        SP.conv_table(bad.to(cuda), bad.to(cuda), 2, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])


def test_layers_reference_golden(cuda):
    """SparseConv3d / SparseInverseConv3d / SubMConv3d modules against the outputs of the reference's own spconv layers"""
    from sst_b200 import spconv_modules as SP
    z = np.load(os.path.join(G, "spconv_layers.npz"))
    feats, coors, shape = torch.from_numpy(z["l_feats"]).to(cuda), torch.from_numpy(z["l_coors"]).to(cuda), z["l_shape"].tolist()
    with torch.no_grad():
        for name in "abc":
            cfg = z[f"conv_{name}_cfg"].tolist()
            conv = SP.SparseConv3d(8, 12, cfg[0:3], stride=cfg[3:6], padding=cfg[6:9], bias=False, indice_key="k").to(cuda)
            inv = SP.SparseInverseConv3d(12, 8, cfg[0:3], indice_key="k", bias=False).to(cuda)
            conv.weight.copy_(torch.from_numpy(z[f"conv_{name}_w"]))
            inv.weight.copy_(torch.from_numpy(z[f"inv_{name}_w"]))
            y = conv(SP.SparseConvTensor(feats, coors, shape, 2))
            assert y.spatial_shape == z[f"conv_{name}_shape"].tolist()
            assert torch.equal(y.indices.cpu(), torch.from_numpy(z[f"conv_{name}_coors"]).int())   # lexicographic order
            _close(y.features, torch.from_numpy(z[f"conv_{name}_out"]), 1e-4)
            back = inv(y)
            assert torch.equal(back.indices, coors) and back.spatial_shape == shape
            _close(back.features, torch.from_numpy(z[f"inv_{name}_out"]), 1e-4)
        sub = SP.SubMConv3d(8, 12, 3, padding=0, bias=True, indice_key="s").to(cuda)
        sub.weight.copy_(torch.from_numpy(z["subm_w"]))
        sub.bias.copy_(torch.from_numpy(z["subm_b"]))
        y = sub(SP.SparseConvTensor(feats, coors, shape, 2))
        _close(y.features, torch.from_numpy(z["subm_out"]), 1e-4)


def _load_sd(net, z, prefix):
    sd = {k[len(prefix):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(prefix)}
    missing, unexpected = net.load_state_dict(sd, strict=True)
    return net


def test_unet_and_mixer_reference_golden(cuda):
    """SimpleSparseUNet / VirtualVoxelMixer (registered names, reference state-dict keys) against the reference classes' outputs;
    eval mode = the fused conv + BN (+ residual) + ReLU launches"""
    from sst_b200 import registry
    z = np.load(os.path.join(G, "spconv_unet.npz"))
    net = registry.MODELS.build(dict(type="SimpleSparseUNet", **SO.SP_UNET, return_multiscale_features=True))
    net = _load_sd(net, z, "unet_sd.").to(cuda).eval()
    feats, coors = torch.from_numpy(z["unet_feats"]).to(cuda), torch.from_numpy(z["unet_coors"]).to(cuda)
    with torch.no_grad():
        out = net(dict(voxel_feats=feats, voxel_coors=coors))[0]
    assert torch.equal(out["voxel_coors"], coors) and out["batch_size"] == 2 and list(out["sparse_shape"]) == SO.SP_UNET["sparse_shape"]
    _close(out["voxel_feats"], torch.from_numpy(z["unet_out"]), 1e-4)
    assert len(out["decoder_features"]) == 4
    for i, d in enumerate(out["decoder_features"]):
        f, c = _sorted(d.features.cpu(), d.indices.cpu())
        assert torch.equal(c, torch.from_numpy(z[f"unet_ms{i}_c"]).int())
        _close(f, torch.from_numpy(z[f"unet_ms{i}_f"]), 1e-4)
    mix = registry.MODELS.build(dict(type="VirtualVoxelMixer", **SO.SP_MIXER))
    mix = _load_sd(mix, z, "mixer_sd.").to(cuda).eval()
    with torch.no_grad():
        f, c, shape = mix(torch.from_numpy(z["mixer_feats"]).to(cuda), torch.from_numpy(z["mixer_coors"]).to(cuda), 3)
    assert torch.equal(c.cpu(), torch.from_numpy(z["mixer_coors"]).int()) and list(shape) == SO.SP_MIXER["sparse_shape"]
    _close(f, torch.from_numpy(z["mixer_out"]), 1e-4)
    # the unfused composition (conv launch, torch BatchNorm1d, activation, torch residual add) gives the same numbers
    from sst_b200 import spconv_modules as SP
    SP.FUSE_EPILOGUE = False
    try:
        with torch.no_grad():
            out2 = net(dict(voxel_feats=feats, voxel_coors=coors))[0]
    finally:
        SP.FUSE_EPILOGUE = True
    _close(out2["voxel_feats"], out["voxel_feats"], 1e-5)


@pytest.mark.parametrize("cin,cout", [(64, 64), (128, 64), (64, 128), (256, 256), (512, 256)])
def test_conv_epilogue_both_precisions(cuda, cin, cout):
    """one launch = gather-GEMM + scale/shift + residual + ReLU; FFMA path and wgmma path against the fp64 table oracle"""
    from sst_b200 import spconv_modules as SP
    shape = [6, 24, 24]
    feats, coors = SO.synth_sparse(cin + cout, 2, shape, 450, cin)
    g = torch.Generator().manual_seed(cin * 7 + cout)
    w = torch.randn((27, cin, cout), generator=g) / (27 * cin) ** 0.5 * 2
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.3
    nbr_ref = SO.neighbour_table(coors, coors, 2, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
    res = torch.randn((coors.shape[0], cout), generator=g)
    nbr, _ = SP.conv_table(coors.to(cuda), coors.to(cuda), 2, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
    for relu, use_res, use_aff in ((True, True, True), (False, False, False)):
        ref = SO.indice_conv(feats, nbr_ref, w, scale if use_aff else None, shift if use_aff else None, res if use_res else None, relu)
        for prec, tol in (("fp32", 1e-4), ("bf16", 5e-3), ("fp32_tc", 1e-4)):
            out = SP.indice_conv(feats.to(cuda), nbr, w.to(cuda), None, scale.to(cuda) if use_aff else None,
                                 shift.to(cuda) if use_aff else None, res.to(cuda) if use_res else None, relu, prec)
            _close(out, ref, tol)


def test_tensor_path_refuses_unsupported_shapes(cuda):
    from sst_b200 import _lib as L, spconv_modules as SP
    feats, coors = SO.synth_sparse(1, 1, [4, 8, 8], 60, 16)
    nbr, _ = SP.conv_table(coors.to(cuda), coors.to(cuda), 1, [4, 8, 8], [4, 8, 8], [3, 3, 3], [1, 1, 1], [1, 1, 1])
    with pytest.raises(L.SSTB200Error, match="tensor-core path"):
        SP.indice_conv(feats.to(cuda), nbr, torch.randn(27, 16, 16, device=cuda), precision="bf16")
    with pytest.raises(L.SSTB200Error):   # CPU tensors: no fallback
        SP.indice_conv(feats, nbr.cpu(), torch.randn(27, 16, 16))


UNET64 = dict(in_channels=64, sparse_shape=[16, 40, 40], norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01), base_channels=64,
              output_channels=128, encoder_channels=((64,), (64, 64, 64), (64, 64, 64), (128, 128, 128)),
              encoder_paddings=((1,), (1, 1, 1), (1, 1, 1), ((0, 1, 1), 1, 1)),
              decoder_channels=((128, 128, 64), (64, 64, 64), (64, 64, 64), (64, 64, 64)), decoder_paddings=((1, 1), (1, 0), (0, 0), (0, 1)))


def _live_init(net, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.2)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.2)
        for p in net.parameters():
            if p.dim() == 5:
                p.mul_(2.0)


def test_unet_fsd_channels_both_precisions(cuda):
    """a SimpleSparseUNet with the channel widths of configs/fsd (64 / 128) against the oracle: fp32 path 1e-4, wgmma path 1e-2"""
    from sst_b200 import registry, spconv_modules as SP
    torch.manual_seed(11)
    net = registry.MODELS.build(dict(type="SimpleSparseUNet", **UNET64)).eval()
    _live_init(net, 13)
    feats, coors = SO.synth_sparse(17, 2, UNET64["sparse_shape"], 900, 64)
    ref, rc = SO.sparse_unet_forward(net.state_dict(), feats, coors, 2, UNET64["sparse_shape"], UNET64["encoder_channels"],
                                     UNET64["encoder_paddings"], UNET64["decoder_channels"], UNET64["decoder_paddings"])
    net = net.to(cuda)
    with torch.no_grad():
        for prec, tol in (("fp32", 1e-4), ("bf16", 1e-2), ("fp32_tc", 1e-4)):
            SP.set_spconv_precision(net, prec)
            out = net(dict(voxel_feats=feats.to(cuda), voxel_coors=coors.to(cuda)))[0]
            assert torch.equal(out["voxel_coors"].cpu(), coors)
            _close(out["voxel_feats"], ref, tol)


def _fsd_scale_input(cuda, n=120000, channels=64):
    """~120k active voxels of a 150k-point sweep on the configs/fsd segmentation grid [32, 640, 640]"""
    from oracle import sst_oracle as O
    pts = O.synth_frame(1000, 150000)
    vs, rng = (0.2, 0.2, 0.2), [-64.0, -64.0, -3.2, 64.0, 64.0, 3.2]
    c = torch.stack([((pts[:, 2] - rng[2]) / vs[2]).floor(), ((pts[:, 1] - rng[1]) / vs[1]).floor(), ((pts[:, 0] - rng[0]) / vs[0]).floor()], 1)
    ok = (c[:, 0] >= 0) & (c[:, 0] < 32) & (c[:, 1] >= 0) & (c[:, 1] < 640) & (c[:, 2] >= 0) & (c[:, 2] < 640)
    c = torch.unique(c[ok].long(), dim=0)
    g = torch.Generator().manual_seed(5)
    c = c[torch.randperm(c.shape[0], generator=g)][:n]
    coors = torch.cat([torch.zeros((c.shape[0], 1), dtype=torch.long), c], 1).int()
    feats = torch.randn((coors.shape[0], channels), generator=g)
    return feats.to(cuda), coors.to(cuda)


def test_full_size_properties(cuda):
    """FSD-size sweep (~100k voxels, grid 32 x 640 x 640): identity kernel, table transposition, fp32 == tensor path, strided
    conv -> inverse conv restores the rows"""
    from sst_b200 import spconv_modules as SP
    feats, coors = _fsd_scale_input(cuda)
    n = coors.shape[0]
    assert n > 60000
    shape = [32, 640, 640]
    nbr, _ = SP.conv_table(coors, coors, 1, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
    assert torch.equal(nbr[:, 13], torch.arange(n, dtype=torch.int32, device=cuda))
    # SubM symmetry: i is o's neighbour at offset k  <=>  o is i's neighbour at offset 26 - k
    o_idx, k_idx = torch.nonzero(nbr >= 0, as_tuple=True)
    assert torch.equal(nbr[nbr[o_idx, k_idx].long(), 26 - k_idx].long(), o_idx)
    w = torch.zeros((27, 64, 64), device=cuda)
    w[13] = torch.eye(64, device=cuda)
    assert torch.equal(SP.indice_conv(feats, nbr, w), feats)                       # identity kernel, fp32 path: exact
    _close(SP.indice_conv(feats, nbr, w, precision="bf16"), feats, 1e-3)            # fp16 operand rounding only
    _close(SP.indice_conv(feats, nbr, w, precision="fp32_tc"), feats, 1e-6)         # split operands: 22 significant bits
    g = torch.Generator().manual_seed(3)
    w = (torch.randn((27, 64, 64), generator=g) / (27 * 64) ** 0.5 * 2).to(cuda)
    a = SP.indice_conv(feats, nbr, w, precision="fp32")
    b = SP.indice_conv(feats, nbr, w, precision="bf16")
    _close(b, a, 5e-3)
    _close(SP.indice_conv(feats, nbr, w, precision="fp32_tc"), a, 1e-4)
    oshape = SO.conv_output_size(shape, [3, 3, 3], [2, 2, 2], [1, 1, 1])
    oc = SP.conv_out_coors(coors, 1, shape, oshape, [3, 3, 3], [2, 2, 2], [1, 1, 1])
    key = (oc[:, 1].long() * oshape[1] + oc[:, 2]) * oshape[2] + oc[:, 3]
    assert bool((key[1:] > key[:-1]).all())                                        # sorted and unique
    down, up = SP.conv_table(coors, oc, 1, shape, oshape, [3, 3, 3], [2, 2, 2], [1, 1, 1], want_nbr=True, want_inv=True)
    o_idx, k_idx = torch.nonzero(down >= 0, as_tuple=True)
    assert torch.equal(up[down[o_idx, k_idx].long(), k_idx].long(), o_idx)          # transposed table = same pairs
    assert int((up >= 0).sum()) == int((down >= 0).sum())
    assert bool((up >= 0).any(1).all())                                            # every input reaches an output (padding 1)


def test_vs_reference_cuda_spconv(cuda):
    """the reference's own CUDA spconv v1 kernels (oracle/_ref, built from mmdet3d/ops/spconv/src unmodified) on the same device tensors at
    the FSD size: index pairs hold the same (input, output) coordinate pairs, features agree; prints both timings"""
    from oracle import build_ref
    from sst_b200 import spconv_modules as SP
    ext = build_ref.load_module("sparse_conv_ext_ref")
    if ext is None:
        pytest.skip("oracle/_ref/sparse_conv_ext_ref*.so not built")
    feats, coors = _fsd_scale_input(cuda)
    shape = [32, 640, 640]
    g = torch.Generator().manual_seed(9)
    w = (torch.randn((3, 3, 3, 64, 64), generator=g) / (27 * 64) ** 0.5 * 2).to(cuda)

    def timed(fn, reps=5):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            r = fn()
        e1.record()
        torch.cuda.synchronize()
        return r, e0.elapsed_time(e1) / reps * 1e3

    try:
        (outids, pairs, num), t_ref_pairs = timed(lambda: ext.get_indice_pairs_3d(coors, 1, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1],
                                                                                   [1, 1, 1], [0, 0, 0], 1, 0))
        ref, t_ref_conv = timed(lambda: ext.indice_conv_fp32(feats, w, pairs, num, coors.shape[0], 0, 1))
    except Exception as e:   # the 2019 kernels are not guaranteed to run on sm_90a / this torch
        pytest.skip(f"reference CUDA spconv did not run here: {type(e).__name__}: {e}")
    (nbr, _), t_tab = timed(lambda: SP.conv_table(coors, coors, 1, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1]))
    w27 = w.reshape(27, 64, 64)
    out32, t32 = timed(lambda: SP.indice_conv(feats, nbr, w27, precision="fp32"))
    w16 = w27.permute(0, 2, 1).contiguous().half()
    out16, t16 = timed(lambda: SP.indice_conv(feats, nbr, w27, w16, precision="bf16"))
    pairs_ref, pairs_here = int(num.sum()), int((nbr >= 0).sum())
    _close(out32, ref, 1e-4)
    _close(out16, ref, 5e-3)
    print(f"\n[spconv SubM 3x3x3 64->64, {coors.shape[0]} voxels, pairs {pairs_ref} / {pairs_here}] reference CUDA: pairs {t_ref_pairs:.0f} us + conv {t_ref_conv:.0f} us | "
          f"sst_b200: table {t_tab:.0f} us + conv fp32 {t32:.0f} us / wgmma {t16:.0f} us")


def _gclose(a, b, tol):
    a, b = a.float().cpu(), b.float().cpu()
    torch.testing.assert_close(a, b, rtol=tol, atol=(tol + 1e-7) * float(b.abs().max()))


@pytest.mark.parametrize("probe_scale", [1.0, 2.0 ** -20], ids=["probe_x1", "probe_x2^-20"])
@pytest.mark.parametrize("cin,cmid,prec,tol", [(8, 12, "fp32", 2e-4), (64, 128, "fp32", 2e-4), (64, 128, "bf16", 1e-2), (64, 128, "fp32_tc", 2e-4)])
def test_layer_gradients(cuda, cin, cmid, prec, tol, probe_scale):
    """SubM -> strided conv -> inverse conv: input and weight gradients (dX = the forward kernel on the transposed table with W^T,
    dW = spconv_dw_kernel) against autograd through the oracle's dense restatement.  probe x 2^-20: the gradient magnitudes of a
    mean-reduced loss, far below what an fp16 operand holds unscaled; the tolerances are the same"""
    from sst_b200 import spconv_modules as SP
    shape = [9, 20, 24]
    feats, coors = SO.synth_sparse(41, 2, shape, 400, cin)
    torch.manual_seed(5)
    sub = SP.SubMConv3d(cin, cmid, 3, padding=1, bias=True, indice_key="s")
    conv = SP.SparseConv3d(cmid, cmid, 3, stride=2, padding=(0, 1, 1), bias=False, indice_key="k")
    inv = SP.SparseInverseConv3d(cmid, cin, 3, indice_key="k", bias=False)
    # oracle (CPU, dense, differentiable)
    ws = [p.detach().clone().requires_grad_(True) for p in (sub.weight, sub.bias, conv.weight, inv.weight)]
    x_ref = feats.clone().requires_grad_(True)
    y = SO.subm_conv(x_ref, coors, 2, shape, ws[0], ws[1])
    y2, oc, oshape = SO.sparse_conv(y, coors, 2, shape, ws[2], [2, 2, 2], [0, 1, 1])
    z_ref = SO.inverse_conv(y2, oc, 2, oshape, coors, shape, ws[3], [2, 2, 2], [0, 1, 1])
    probe = torch.randn(z_ref.shape, generator=torch.Generator().manual_seed(1)) * probe_scale
    (z_ref * probe).sum().backward()
    for m in (sub, conv, inv):
        m.to(cuda)
        m.precision = prec
    x = feats.to(cuda).requires_grad_(True)
    z = inv(conv(sub(SP.SparseConvTensor(x, coors.to(cuda), shape, 2))))
    _gclose(z.features.detach(), z_ref.detach(), tol)
    (z.features * probe.to(cuda)).sum().backward()
    _gclose(x.grad, x_ref.grad, tol)
    for p, r in zip((sub.weight, sub.bias, conv.weight, inv.weight), ws):
        _gclose(p.grad, r.grad, tol)


def test_unet_gradients(cuda):
    """SimpleSparseUNet with gradients enabled (frozen BatchNorm statistics): the loss gradient w.r.t. the input features and every
    parameter against autograd through the oracle"""
    from sst_b200 import registry
    cfg = dict(SO.SP_UNET)
    torch.manual_seed(2)
    net = registry.MODELS.build(dict(type="SimpleSparseUNet", **cfg)).eval()
    _live_init(net, 4)
    feats, coors = SO.synth_sparse(6, 2, cfg["sparse_shape"], 300, 8)
    sd = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in net.state_dict().items()}
    x_ref = feats.clone().requires_grad_(True)
    ref = SO.sparse_unet_forward(sd, x_ref, coors, 2, cfg["sparse_shape"], cfg["encoder_channels"], cfg["encoder_paddings"], cfg["decoder_channels"],
                                 cfg["decoder_paddings"])[0]
    probe = torch.randn(ref.shape, generator=torch.Generator().manual_seed(9))
    (ref * probe).sum().backward()
    net = net.to(cuda)
    x = feats.to(cuda).requires_grad_(True)
    out = net(dict(voxel_feats=x, voxel_coors=coors.to(cuda)))[0]["voxel_feats"]
    _gclose(out.detach(), ref.detach(), 2e-4)
    (out * probe.to(cuda)).sum().backward()
    _gclose(x.grad, x_ref.grad, 1e-3)
    n = 0
    for name, p in net.named_parameters():
        _gclose(p.grad, sd[name].grad, 1e-3)
        n += 1
    assert n > 60


def test_sparse_unet_dense_branch(cuda):
    """SparseUNet.forward (PartA2's middle encoder, sparse_unet.py:114-165): the detection branch = SparseConv (3,1,1) / stride (2,1,1) on
    the last encoder stage, densified to [N, C*D, H, W]; the segmentation branch = the decoder output"""
    from sst_b200 import registry
    cfg = dict(in_channels=8, sparse_shape=[41, 32, 32], norm_cfg=dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01), base_channels=8,
               output_channels=16, encoder_channels=((8,), (8, 8, 8), (16, 16, 16), (16, 16, 16)),
               encoder_paddings=((1,), (1, 1, 1), (1, 1, 1), ((0, 1, 1), 1, 1)),
               decoder_channels=((16, 16, 16), (16, 16, 8), (8, 8, 8), (8, 8, 8)), decoder_paddings=((1, 0), (1, 0), (0, 0), (0, 1)))
    torch.manual_seed(4)
    net = registry.MODELS.build(dict(type="SparseUNet", **cfg)).eval()
    _live_init(net, 6)
    feats, coors = SO.synth_sparse(12, 2, cfg["sparse_shape"], 600, 8)
    sd = {k: v.float() for k, v in net.state_dict().items()}
    seg_ref, _ = SO.sparse_unet_forward(sd, feats, coors, 2, cfg["sparse_shape"], cfg["encoder_channels"], cfg["encoder_paddings"],
                                        cfg["decoder_channels"], cfg["decoder_paddings"])
    # detection branch from the oracle's pieces: encoder up to the last stage, then conv_out + BN + ReLU, densified
    x = SO._block(SO._T(feats, coors, cfg["sparse_shape"], 2), sd, "conv_input.", "subm", "subm1", 1e-3, padding=1)
    for i, blocks in enumerate(cfg["encoder_channels"]):
        for j in range(len(blocks)):
            pad = tuple(cfg["encoder_paddings"][i])[j]
            p = f"encoder_layers.encoder_layer{i + 1}.{j}."
            x = SO._block(x, sd, p, "conv", f"spconv{i + 1}", 1e-3, stride=2, padding=pad) if (i != 0 and j == 0) else \
                SO._block(x, sd, p, "subm", f"subm{i + 1}", 1e-3, padding=pad)
    y = SO._block(x, sd, "conv_out.", "conv", "spconv_down2", 1e-3, stride=(2, 1, 1), padding=0)
    dense_ref = SO._dense(y.f, y.c, 2, y.shape)
    net = net.to(cuda)
    with torch.no_grad():
        out = net(feats.to(cuda), coors.to(cuda), 2)
    _close(out["seg_features"], seg_ref, 1e-4)
    N, C, D, H, W = dense_ref.shape
    assert list(out["spatial_features"].shape) == [N, C * D, H, W]
    _close(out["spatial_features"], dense_ref.reshape(N, C * D, H, W), 1e-4)
