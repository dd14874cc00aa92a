"""GPU parity: FSD SIR (S1-S3) through the registered modules / C ABI vs the oracle and the reference golden fixture."""
import os

import numpy as np
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu


def _sir(in_ch, feat, nb, seed=0):
    from sst_b200.sir_modules import SIR
    torch.manual_seed(seed)
    m = SIR(num_blocks=nb, in_channels=in_ch, feat_channels=[[feat, feat]] * nb, rel_mlp_hidden_dims=[[16, 32]] * nb,
            norm_cfg=dict(type='LN', eps=1e-3), mode='max', xyz_normalizer=[20, 20, 4], act='gelu', unique_once=True).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if n_.endswith("1.weight") or "norm.weight" in n_ else 0.0))
    return m


def test_sir_golden_fixture(cuda):
    """Weights + inputs + outputs produced by the unmodified reference SIR (tests/golden/sir_small.npz)."""
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "sir_small.npz"))
    m = _sir([32, 37, 37], 32, 3)
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w.")}
    m.load_state_dict(sd, strict=True)
    m = m.to(cuda)
    t = lambda k: torch.from_numpy(z[k]).to(cuda)
    with torch.no_grad():
        a, b, c = m(t("points"), t("feats"), t("coors"), t("f_cluster"))
    assert torch.equal(c.cpu(), torch.from_numpy(z["out_coors"]))
    torch.testing.assert_close(a.cpu(), torch.from_numpy(z["out_point"]), rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(b.cpu(), torch.from_numpy(z["out_group"]), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("N,G", [(20000, 64), (150000, 256), (50, 50)])
def test_sir_config3_parity(cuda, N, G):
    """BASELINE config 3 shape (FSD: Cin 84/133/133, 128-d, rel-MLP 16-32, LN eps 1e-3, GELU, max)."""
    g = torch.Generator().manual_seed(N)
    points = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1)
    feats = torch.randn(N, 79, generator=g)
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1)
    fcl = torch.randn(N, 3, generator=g) * 2
    m = _sir([84, 133, 133], 128, 3)
    ref = O.sir_forward(points, feats, coors, fcl, dict(m.state_dict()), 3, 3, 2, [20, 20, 4])
    m = m.to(cuda)
    with torch.no_grad():
        a, b, c = m(points.to(cuda), feats.to(cuda), coors.to(cuda), fcl.to(cuda))
    assert torch.equal(c.cpu(), ref[2])
    for got, exp in ((a, ref[0]), (b, ref[1])):
        err = (got.cpu() - exp).abs().max().item() / exp.abs().max().item()
        assert err < 1e-3, err


def test_sir_layer_without_f_cluster_and_shortcut(cuda):
    """f_cluster=None (computed from the group mean, voxel_encoder.py:717-723) and the shortcut branch."""
    from sst_b200.sir_modules import SIRLayer
    torch.manual_seed(0)
    N, G, cin = 4000, 30, 35
    m = SIRLayer(in_channels=cin, feat_channels=[32, 32], rel_mlp_hidden_dims=[16, 32], norm_cfg=dict(type='LN', eps=1e-3),
                 mode='max', return_point_feats=True, rel_dist_scaler=10.0, xyz_normalizer=[20, 20, 4], act='gelu').eval()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(N, cin, generator=g)
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([torch.zeros_like(gid), gid], 1)
    new_coors, inv = torch.unique(coors, return_inverse=True, dim=0)
    w = {("x." + k): v for k, v in m.state_dict().items()}
    pf, gf = O.sir_layer_forward(x, inv, new_coors.shape[0], None, w, "x.", 3, 2, [20, 20, 4], 1e-3, "gelu", 10.0)
    m = m.to(cuda)
    with torch.no_grad():
        a, b = m(x.to(cuda), coors.to(cuda))
    torch.testing.assert_close(a.cpu(), pf, rtol=1e-3, atol=1e-4)
    torch.testing.assert_close(b.cpu(), gf, rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("N,G", [(20000, 64), (150000, 256), (300, 7), (129, 1)])
def test_sir_config3_bf16_parity(cuda, N, G):
    """Tensor-core path (wgmma, bf16 operands / fp32 accumulate): 1e-2 of the fp32 oracle (north_star tolerance for bf16);
    group coordinates stay bit-exact.  Also covers the in-place [points || feats] hand-over between blocks."""
    g = torch.Generator().manual_seed(N + 1)
    points = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1)
    feats = torch.randn(N, 79, generator=g)
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1)
    fcl = torch.randn(N, 3, generator=g) * 2
    m = _sir([84, 133, 133], 128, 3)
    ref = O.sir_forward(points, feats, coors, fcl, dict(m.state_dict()), 3, 3, 2, [20, 20, 4])
    m = m.to(cuda)
    m.precision = "bf16"
    with torch.no_grad():
        a, b, c = m(points.to(cuda), feats.to(cuda), coors.to(cuda), fcl.to(cuda))
    assert torch.equal(c.cpu(), ref[2])
    for got, exp in ((a, ref[0]), (b, ref[1])):
        assert torch.isfinite(got).all()
        err = (got.cpu() - exp).abs().max().item() / exp.abs().max().item()
        assert err < 1e-2, err


def test_sir_bf16_unsupported_shape_fails_loudly(cuda):
    from sst_b200._lib import SSTB200Error
    m = _sir([32, 37, 37], 32, 3).to(cuda)
    m.precision = "bf16"
    N = 100
    with pytest.raises(SSTB200Error), torch.no_grad():
        m(torch.randn(N, 5, device=cuda), torch.randn(N, 27, device=cuda), torch.zeros(N, 3, dtype=torch.long, device=cuda),
          torch.randn(N, 3, device=cuda))


@pytest.mark.parametrize("N,G", [(150000, 256), (5000, 5000), (1000, 1), (77, 9000)])
def test_group_csr(cuda, N, G):
    """offsets = exclusive scan of the group sizes; order = a permutation grouping the points (small-G and large-G kernels)."""
    from sst_b200.sir_modules import group_csr
    g = torch.Generator().manual_seed(G)
    inv = torch.randint(0, G, (N,), generator=g)
    off, order = group_csr(inv.to(cuda), G)
    off, order = off.cpu().long(), order.cpu().long()
    cnt = torch.bincount(inv, minlength=G)
    assert torch.equal(off, torch.cat([torch.zeros(1, dtype=torch.long), cnt.cumsum(0)]))
    assert torch.equal(order.sort().values, torch.arange(N))
    assert torch.equal(inv[order], inv.sort().values)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sir_empty_input(cuda, precision):
    """No points: shapes are kept, nothing is launched (the reference returns empty tensors through torch.unique / scatter)."""
    m = _sir([84, 133, 133], 128, 3).to(cuda)
    m.precision = precision
    with torch.no_grad():
        a, b, c = m(torch.zeros(0, 5, device=cuda), torch.zeros(0, 79, device=cuda), torch.zeros(0, 3, dtype=torch.long, device=cuda),
                    torch.zeros(0, 3, device=cuda))
    assert a.shape == (0, 128) and b.shape == (0, 768) and c.shape == (0, 3)


def test_sir_training_gradients(cuda):
    """SIR with gradients enabled (composition over the segmented-reduction forward / backward kernels): outputs, the feature gradient and
    every parameter gradient against autograd through the oracle (pinned to the reference's autograd)"""
    m = _sir([20, 37, 37], 32, 3).train()
    g = torch.Generator().manual_seed(1)
    N, G = 3000, 60
    points = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1)
    feats = torch.randn(N, 15, generator=g)
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1)
    fcl = torch.randn(N, 3, generator=g) * 2
    w = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    f_ref = feats.clone().requires_grad_(True)
    ref = O.sir_forward(points, f_ref, coors, fcl, w, 3, 3, 2, [20, 20, 4])
    (ref[0].square().sum() + ref[1].square().sum()).backward()
    m = m.to(cuda)
    f = feats.to(cuda).requires_grad_(True)
    a, b, c = m(points.to(cuda), f, coors.to(cuda), fcl.to(cuda))
    assert torch.equal(c.cpu(), ref[2])
    torch.testing.assert_close(a.detach().cpu(), ref[0].detach(), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(b.detach().cpu(), ref[1].detach(), rtol=1e-4, atol=1e-4)
    (a.square().sum() + b.square().sum()).backward()
    torch.testing.assert_close(f.grad.cpu(), f_ref.grad, rtol=1e-3, atol=1e-4 * float(f_ref.grad.abs().max()))
    for name, p in m.named_parameters():
        torch.testing.assert_close(p.grad.cpu(), w[name].grad, rtol=1e-3, atol=2e-4 * float(w[name].grad.abs().max()) + 1e-7)
