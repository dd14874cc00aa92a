"""CPU, build container only: autograd through oracle.sir_layer_forward against the reference's own SIRLayer on the cases the SIR
training kernels are checked on beyond test_oracle_sir_gradients_match_reference - the f_cluster gradient, f_cluster=None, the
RoI-head layer shape (rel_mlp_in_channel=13, return_point_feats=True) and act='relu'.  Skipped where the reference tree is absent."""
import pytest
import torch

from oracle import ref_shim, sst_oracle as O

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")

CASES = {
    "f_cluster_grad": dict(cin=35, feats=[32, 32], rel_in=3, act="gelu", fcl=True),
    "f_cluster_none": dict(cin=35, feats=[32, 32], rel_in=3, act="gelu", fcl=False),
    "roi_head": dict(cin=213, feats=[128, 128], rel_in=13, act="gelu", fcl=True),
    "relu": dict(cin=35, feats=[32, 32], rel_in=3, act="relu", fcl=True),
}


@pytest.fixture(scope="module")
def R():
    return ref_shim.load()


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_sir_layer_grads_match_reference(R, case):
    k = CASES[case]
    torch.manual_seed(3)
    N, G = 1500, 37
    g = torch.Generator().manual_seed(4)
    x = torch.randn(N, k["cin"], generator=g)
    x[:, :3] *= 10
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([torch.zeros_like(gid), gid], 1)
    fcl = torch.randn(N, k["rel_in"], generator=g) * 2 if k["fcl"] else None
    m = R.SIRLayer(in_channels=k["cin"], feat_channels=list(k["feats"]), rel_mlp_hidden_dims=[16, 32], rel_mlp_in_channel=k["rel_in"],
                   norm_cfg=dict(type='LN', eps=1e-3), mode='max', return_point_feats=True, rel_dist_scaler=10.0,
                   xyz_normalizer=[20, 20, 4], act=k["act"]).train()
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if n_.endswith("1.weight") or "norm.weight" in n_ else 0.0))
    probe_p, probe_g = torch.randn(N, k["feats"][-1], generator=g), torch.randn(G, sum(k["feats"]), generator=g)

    x_r = x.clone().requires_grad_(True)
    f_r = fcl.clone().requires_grad_(True) if fcl is not None else None
    pf_r, gf_r = m(x_r, coors, f_r)
    ((pf_r * probe_p).sum() + (gf_r * probe_g).sum()).backward()

    _, inv = torch.unique(coors, return_inverse=True, dim=0)
    w = {"x." + n_: v.detach().clone().requires_grad_(True) for n_, v in m.state_dict().items()}
    x_o = x.clone().requires_grad_(True)
    f_o = fcl.clone().requires_grad_(True) if fcl is not None else None
    pf_o, gf_o = O.sir_layer_forward(x_o, inv, G, f_o, w, "x.", 3, 2, [20, 20, 4], 1e-3, k["act"], 10.0)
    ((pf_o * probe_p).sum() + (gf_o * probe_g).sum()).backward()

    torch.testing.assert_close(pf_o, pf_r, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(gf_o, gf_r, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(x_o.grad, x_r.grad, rtol=1e-4, atol=1e-6)
    if fcl is not None:
        torch.testing.assert_close(f_o.grad, f_r.grad, rtol=1e-4, atol=1e-6)
    for n_, p in m.named_parameters():  # fp32 sums over 1500 points on both sides: tolerance relative to the largest entry
        torch.testing.assert_close(w["x." + n_].grad, p.grad, rtol=2e-4, atol=1e-5 * float(p.grad.abs().max()), msg=n_)
