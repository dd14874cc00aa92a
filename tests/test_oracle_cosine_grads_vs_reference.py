"""CPU, build container only: autograd through the oracle's cosine attention (oracle.sst_oracle.multihead_attention(cosine=True))
against autograd through the reference's own SSTv2 with layer_cfg cosine - the checker that tests/test_gpu_train_cosine.py trusts.
Skipped where /root/reference does not exist (e.g. the GPU box)."""
import pytest
import torch

from oracle import ref_shim, sst_oracle as O

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}
TAU_MIN = 0.2


@pytest.fixture(scope="module")
def R():
    return ref_shim.load()


# per-layer temperatures: shared (one value per layer) or per head, with a head below tau_min (clamped: no gradient) and one
# exactly at tau_min (the clamp passes the gradient at equality)
TAUS = {
    "shared_above": (False, [[0.5], [0.35]]),
    "shared_at_min": (False, [[TAU_MIN], [0.3]]),
    "per_head": (True, [[0.1, TAU_MIN, 0.25, 0.4, 0.6, 0.8, 1.0, 0.3], [0.9, 0.15, TAU_MIN, 0.5, 0.22, 0.7, 0.33, 1.0]]),
}


@pytest.mark.parametrize("case", sorted(TAUS))
def test_oracle_cosine_gradients_match_reference(R, case):
    non_shared, taus = TAUS[case]
    lc = dict(cosine=True, tau_min=TAU_MIN, non_shared_tau=non_shared)
    torch.manual_seed(0)
    pts = O.synth_frame(1000, 6000)
    coors = torch.nn.functional.pad(torch.unique(O.dynamic_voxelize(pts, VS, RNG), dim=0), (1, 0), value=0)
    g = torch.Generator().manual_seed(1)
    feats = torch.randn(coors.shape[0], 128, generator=g)
    il = R.SSTInputLayerV2(DROP_TEST, (12, 12, 1), (468, 468, 1), shuffle_voxels=False, debug=True, mute=True).eval()
    bb = R.SSTv2(d_model=[128], nhead=[8], num_blocks=1, dim_feedforward=[256], output_shape=[468, 468], num_attached_conv=0,
                 to_bev=False, layer_cfg=lc).eval()
    with torch.no_grad():
        for n_, p in bb.named_parameters():
            if n_.endswith("tau"):
                p.copy_(torch.tensor(taus[int(n_.split("encoder_list.")[1][0])]).view(p.shape))
            elif p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
    x_r = feats.clone().requires_grad_(True)
    out_r = bb(il(x_r, coors, 1))[0]["voxel_feats"]
    probe = torch.randn(out_r.shape, generator=torch.Generator().manual_seed(2))
    (out_r * probe).sum().backward()

    w = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in bb.state_dict().items()}
    x_o = feats.clone().requires_grad_(True)
    info_o = O.input_layer_v2(x_o, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    out_o = O.sstv2_forward(info_o, w, [8], 1, layer_cfg=lc)
    torch.testing.assert_close(out_o, out_r, rtol=1e-5, atol=1e-5)
    (out_o * probe).sum().backward()
    torch.testing.assert_close(x_o.grad, x_r.grad, rtol=2e-4, atol=1e-6 * float(x_r.grad.abs().max()))
    taus_seen = 0
    for k, p in bb.named_parameters():
        # atol: fp32 summation-order noise on the largest entry (elementwise rtol alone fails on entries near zero)
        torch.testing.assert_close(w[k].grad, p.grad, rtol=2e-4, atol=1e-6 * float(p.grad.abs().max()), msg=k)
        if k.endswith("tau"):
            taus_seen += 1
            below = p.detach().view(-1) < TAU_MIN
            assert torch.all(p.grad.view(-1)[below] == 0) and torch.all(w[k].grad.view(-1)[below] == 0), k
            at = p.detach().view(-1) == TAU_MIN
            assert torch.all(w[k].grad.view(-1)[at] != 0), k
    assert taus_seen == 2
