"""GPU: training path with cosine attention (logits = normalize(q) . normalize(k) / clamp(tau, tau_min), models/sst/cosine_msa.py)
- gradients of csrc/sra_train.cu through sst_b200.train against autograd through the CPU oracle, which
tests/test_oracle_cosine_grads_vs_reference.py pins to the reference's own autograd."""
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]
DROP_TEST = {0: {'max_tokens': 30, 'drop_range': (0, 30)}, 1: {'max_tokens': 60, 'drop_range': (30, 60)},
             2: {'max_tokens': 100, 'drop_range': (60, 100)}, 3: {'max_tokens': 144, 'drop_range': (100, 100000)}}


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _setup(P, num_blocks, layer_cfg, taus=None, seed=0):
    """Voxel features + coordinates of one synthetic frame and a bf16 SSTv2 with `layer_cfg`; taus(layer_index, tau) -> new tau."""
    from sst_b200.sst_modules import SSTInputLayerV2, SSTv2
    p = O.synth_frame(900 + seed, P)
    c = torch.unique(O.dynamic_voxelize(p, VS, RNG), dim=0)
    coors = torch.nn.functional.pad(c, (1, 0), value=0).int()
    g = torch.Generator().manual_seed(seed)
    feats = torch.randn(coors.shape[0], 128, generator=g)
    torch.manual_seed(seed)
    bb = SSTv2(d_model=[128] * num_blocks, nhead=[8] * num_blocks, num_blocks=num_blocks, dim_feedforward=[256] * num_blocks,
               output_shape=[468, 468], num_attached_conv=0, to_bev=False, precision="bf16", layer_cfg=layer_cfg)
    with torch.no_grad():
        li = 0
        for n_, q in bb.named_parameters():
            if n_.endswith("tau"):
                if taus is not None:
                    q.copy_(taus(li, q))
                li += 1
            elif q.dim() == 1:
                q.copy_(torch.randn(q.shape, generator=g) * 0.1 + (1.0 if "norm" in n_ and "weight" in n_ else 0.0))
    il = SSTInputLayerV2(DROP_TEST, (12, 12, 1), (468, 468, 1), shuffle_voxels=False, mute=True)
    return feats, coors, il, bb


def _oracle_weights(module):
    """Leaf copies of `module`'s state for autograd through the oracle.  A shared tau enters as 8 equal per-head copies, so the
    oracle also yields every head's share of its gradient (the shared gradient is their sum)."""
    return {k: (v.detach().reshape(-1)[:1].expand(1, 8, 1, 1).clone() if k.endswith("tau") and v.numel() == 1 else v.detach().clone())
            .requires_grad_(True) for k, v in module.state_dict().items()}


def _tau_err(got, ref_heads):
    """|d tau error| relative to the layer's d tau scale.  Per-head tau: the largest |d tau| of the layer.  Shared tau: its gradient is
    the sum of the eight heads' shares, which can cancel to a small fraction of them, so the scale is the sum of the shares' magnitudes
    (the size of the addends that carry the bf16 rounding)."""
    ref_heads = ref_heads.reshape(-1)
    if got.numel() == ref_heads.numel():
        return (got.reshape(-1) - ref_heads).abs().max().item() / ref_heads.abs().max().item()
    return abs(got.reshape(-1)[0].item() - ref_heads.sum().item()) / ref_heads.abs().sum().item()


def _stack_grads(cuda, P, num_blocks, layer_cfg, taus):
    """(oracle weights with .grad, oracle input grad, CUDA module after backward, CUDA input grad, forward rel err)."""
    feats, coors, il, bb = _setup(P, num_blocks, layer_cfg, taus)
    w = _oracle_weights(bb)
    xo = feats.clone().requires_grad_(True)
    info_o = O.input_layer_v2(xo, coors, DROP_TEST, (12, 12, 1), (468, 468, 1))
    yo = O.sstv2_forward(info_o, w, [8] * num_blocks, num_blocks, layer_cfg=layer_cfg)
    gy = torch.randn(yo.shape, generator=torch.Generator().manual_seed(5)) / yo.shape[0]
    (yo * gy).sum().backward()
    bb = bb.to(cuda).train()
    xg = feats.to(cuda).requires_grad_(True)
    info = il.train()(xg, coors.to(cuda), 1)
    yg = bb(info)[0]["voxel_feats"]
    fwd_err = _rel(yg.detach().cpu(), yo.detach())
    (yg * gy.to(cuda)).sum().backward()
    return w, xo.grad, bb, xg.grad.cpu(), fwd_err


def _uniform_taus(li, q):
    """tau ~ U[0.1, 1] per element (per head with non_shared_tau), seeded per layer."""
    return torch.rand(q.shape, generator=torch.Generator().manual_seed(100 + li)) * 0.9 + 0.1


@pytest.mark.parametrize("non_shared", [False, True], ids=["shared_tau", "per_head_tau"])
@pytest.mark.parametrize("P,num_blocks", [(20000, 1), (60000, 2)])
def test_cosine_stack_gradients_match_oracle_autograd(cuda, P, num_blocks, non_shared):
    lc = dict(cosine=True, tau_min=0.01, non_shared_tau=non_shared)
    w, gxo, bb, gx, fwd_err = _stack_grads(cuda, P, num_blocks, lc, _uniform_taus)
    assert fwd_err < 1e-2, f"training forward rel err {fwd_err}"
    assert _rel(gx, gxo) < 2e-2, f"d input: {_rel(gx, gxo)}"
    bad, taus = {}, 0
    for name, p in bb.named_parameters():
        assert p.grad is not None, name
        ref = w[name].grad
        if name.endswith("tau"):
            taus += 1
            assert p.grad.shape == p.shape and p.numel() == (8 if non_shared else 1)
            err = _tau_err(p.grad.cpu(), ref)
            if err > 3e-2:
                bad[name] = err
        elif _rel(p.grad.cpu(), ref) > 2e-2:
            bad[name] = _rel(p.grad.cpu(), ref)
    assert taus == 2 * num_blocks
    assert not bad, f"gradients off (bf16 tolerance 2e-2 of max-abs, tau 3e-2): {bad}"


def test_cosine_tau_gradient_clamp_rule(cuda):
    """tau below tau_min: clamped, gradient exactly 0; tau == tau_min: torch's clamp(min=) passes the gradient."""
    tau_min = 0.2
    vals = [[0.1, 0.2, 0.3, 0.45, 0.6, 0.75, 0.9, 1.0], [0.2, 0.1, 0.25, 0.5, 0.35, 0.8, 0.65, 0.4]]

    def taus(li, q):
        return torch.tensor(vals[li]).view(q.shape)

    lc = dict(cosine=True, tau_min=tau_min, non_shared_tau=True)
    w, _, bb, _, _ = _stack_grads(cuda, 20000, 1, lc, taus)
    for li in range(2):
        name = f"block_list.0.encoder_list.{li}.win_attn.self_attn.tau"
        got = dict(bb.named_parameters())[name].grad.cpu().view(-1)
        ref = w[name].grad.view(-1)
        below, at = vals[li].index(0.1), vals[li].index(0.2)
        assert got[below].item() == 0.0 and ref[below].item() == 0.0
        assert ref[at].item() != 0.0 and got[at].item() != 0.0
        assert abs(got[at].item() - ref[at].item()) < 3e-2 * ref.abs().max().item()


def test_cosine_tau_gradient_is_reproducible(cuda):
    """d tau is reduced in a fixed order (no float atomics): two backward passes agree bit for bit."""
    lc = dict(cosine=True, tau_min=0.01, non_shared_tau=True)
    feats, coors, il, bb = _setup(20000, 1, lc, _uniform_taus)
    bb = bb.to(cuda).train()
    info = il.train()(feats.to(cuda), coors.to(cuda), 1)
    gy = torch.randn(info["voxel_feats"].shape, generator=torch.Generator().manual_seed(5)).to(cuda)
    grads = []
    for _ in range(2):
        bb.zero_grad()
        (bb(info)[0]["voxel_feats"] * gy).sum().backward()
        grads.append([p.grad.clone() for n_, p in bb.named_parameters() if n_.endswith("tau")])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def _centerhead_cfg(num_blocks=4):
    """configs/sst_refactor/sst_waymoD5_1x_3class_centerhead.py: 5-dim points, pos_temperature 1000, cosine attention."""
    from sst_b200 import flagship as fl
    cfg = fl.sst_cfg(num_blocks=num_blocks, in_channels=5)
    cfg["middle_encoder"]["pos_temperature"] = 1000
    cfg["backbone"]["layer_cfg"] = dict(use_bn=False, cosine=True, tau_min=0.01)
    cfg["backbone"]["precision"] = "bf16"
    return cfg


def test_centerhead_full_model_train_step_gradients(cuda):
    """DynamicVFE (training-mode BN) -> SSTInputLayerV2 (training drop_info, shuffle off) -> SSTv2 (4 blocks, cosine): loss and
    every parameter gradient against autograd through the oracle."""
    from sst_b200 import flagship as fl
    vfe, il, bb = fl.build_sst(_centerhead_cfg(), seed=3)
    pts = torch.cat([O.synth_frame(41, 12000, extra_dims=2), O.synth_frame(42, 9000, extra_dims=2)])
    c3 = O.dynamic_voxelize(pts, VS, RNG)
    coors = torch.cat([torch.nn.functional.pad(c3[:12000], (1, 0), value=0), torch.nn.functional.pad(c3[12000:], (1, 0), value=1)])
    lc = dict(use_bn=False, cosine=True, tau_min=0.01)
    wv = {k: v.detach().clone().requires_grad_(k in dict(vfe.named_parameters())) for k, v in vfe.state_dict().items()}
    wb = _oracle_weights(bb)
    vf_o, vc_o = O.dynamic_vfe_forward(pts, coors, wv, VS, RNG, 2, training=True)
    info_o = O.input_layer_v2(vf_o, vc_o, fl.DROP_TRAIN, (12, 12, 1), (468, 468, 1), pos_temperature=1000)
    out_o = O.sstv2_forward(info_o, wb, [8] * 4, 4, layer_cfg=lc)
    loss_o = out_o.square().mean()
    loss_o.backward()
    vfe, bb = vfe.to(cuda).train(), bb.to(cuda).train()
    il.train()
    il.shuffle_voxels = False
    vf, vc = vfe(pts.to(cuda), coors.to(cuda))
    assert torch.equal(vc.cpu().long(), vc_o.long())
    info = il(vf, vc, 2)
    assert torch.equal(info["voxel_keep_inds"].cpu(), info_o["voxel_keep_inds"])
    loss = bb(info)[0]["voxel_feats"].float().square().mean()
    loss.backward()
    assert abs(loss.item() - loss_o.item()) < 2e-2 * abs(loss_o.item())
    bad, taus = {}, 0
    for name, p in list(vfe.named_parameters()) + list(bb.named_parameters()):
        ref = (wv if name.startswith("vfe_layers") else wb)[name].grad
        taus += name.endswith("tau")
        r = _tau_err(p.grad.cpu(), ref) if name.endswith("tau") else _rel(p.grad.cpu(), ref)
        if r > 3e-2:
            bad[name] = r
    assert taus == 8
    assert not bad, bad


def test_cosine_training_loop(cuda):
    """Ten TrainStep steps on a fixed frame: the loss goes down, the parameters stay finite, and every layer's tau is updated -
    tau is a backbone parameter, so it lives in FlatAdamW's flat buffer and is covered by the one all-reduce."""
    from sst_b200 import flagship as fl
    from sst_b200.train import TrainStep
    vfe, il, bb = fl.build_sst(_centerhead_cfg(), seed=0)
    ts = TrainStep(vfe.to(cuda), il, bb.to(cuda), fl.VOXEL_SIZE, fl.PC_RANGE, lr=1e-3)
    flat = ts.opt.flat
    taus = [p for n_, p in bb.named_parameters() if n_.endswith("tau")]
    assert len(taus) == 8
    for p in ts.opt.params:   # one-element taus are padded, so every view stays 16-byte aligned for the kernels' vector loads
        assert p.data_ptr() % 16 == 0 and p.grad.data_ptr() % 16 == 0
    for t in taus:   # views into the flat parameter / gradient buffers
        assert flat.data_ptr() <= t.data_ptr() < flat.data_ptr() + flat.numel() * 4
        assert ts.opt.flat_grad.data_ptr() <= t.grad.data_ptr() < ts.opt.flat_grad.data_ptr() + flat.numel() * 4
    tau0 = [t.detach().clone() for t in taus]
    frame = [fl.synth_frame(7, 30000, extra_dims=2).to(cuda)]
    losses = [ts.step(frame).item() for _ in range(11)]
    assert losses[10] < losses[0], losses
    for n_, p in list(vfe.named_parameters()) + list(bb.named_parameters()):
        assert torch.isfinite(p).all(), n_
    for t, t0 in zip(taus, tau0):
        assert not torch.equal(t.detach(), t0)


def test_batchnorm_training_still_refused(cuda):
    from sst_b200._lib import SSTB200Error
    feats, coors, il, bb = _setup(20000, 1, dict(use_bn=True, cosine=True))
    bb = bb.to(cuda).train()
    xg = feats.to(cuda).requires_grad_(True)
    info = il.train()(xg, coors.to(cuda), 1)
    with pytest.raises(SSTB200Error, match="LayerNorm"):
        bb(info)
