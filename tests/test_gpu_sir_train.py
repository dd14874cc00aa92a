"""GPU: SIR / SIRLayer training through the native fp32 forward-with-state and backward (SirLayerFunction), against float64
autograd through the oracle (pinned to the reference's autograd by the CPU oracle tests), and at config scale against the composed
torch path.  Error = max |diff| / max |ref| per tensor."""
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

TOL = 1e-3
NZ = [20, 20, 4]


def _rel(got, ref):
    ref = ref.detach().double().cpu()
    return (got.detach().double().cpu() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _init(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n_, p in m.named_parameters():
            if p.dim() == 1:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + (1.0 if n_.endswith("1.weight") or "norm.weight" in n_ else 0.0))
    return m


def _sir(in_ch, feat, nb, act="gelu", seed=0):
    from sst_b200.sir_modules import SIR
    torch.manual_seed(seed)
    m = SIR(num_blocks=nb, in_channels=in_ch, feat_channels=[[feat, feat]] * nb, rel_mlp_hidden_dims=[[16, 32]] * nb,
            norm_cfg=dict(type='LN', eps=1e-3), mode='max', xyz_normalizer=NZ, act=act, unique_once=True)
    return _init(m, seed + 1).train()


def _layer(cin, feats, rel_in=3, act="gelu", seed=0, **kw):
    from sst_b200.sir_modules import SIRLayer
    torch.manual_seed(seed)
    m = SIRLayer(in_channels=cin, feat_channels=feats, rel_mlp_hidden_dims=[16, 32], rel_mlp_in_channel=rel_in,
                 norm_cfg=dict(type='LN', eps=1e-3), mode='max', return_point_feats=True, rel_dist_scaler=10.0, xyz_normalizer=NZ,
                 act=act, **kw)
    return _init(m, seed + 1).train()


def _frame(N, G, nfeat, seed):
    g = torch.Generator().manual_seed(seed)
    points = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1)
    feats = torch.randn(N, nfeat, generator=g)
    gid = torch.randint(0, G, (N,), generator=g)
    gid[:G] = torch.arange(G)[:N]  # every group occupied
    coors = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1)
    fcl = torch.randn(N, 3, generator=g) * 2
    return points, feats, coors, fcl, g


@pytest.mark.parametrize("N,G", [(20000, 64), (3000, 60), (129, 1), (50, 50)])
def test_sir_fsd_dims_vs_fp64_oracle(cuda, N, G):
    """SIR, 3 blocks at FSD dims (84/133/133, [128, 128], rel [16, 32], GELU): outputs, grad feats, grad f_cluster, every parameter."""
    points, feats, coors, fcl, g = _frame(N, G, 79, N + G)
    m = _sir([84, 133, 133], 128, 3)
    w = {k: v.detach().double().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    f_o, c_o = feats.double().requires_grad_(True), fcl.double().requires_grad_(True)
    ref = O.sir_forward(points.double(), f_o, coors, c_o, w, 3, 3, 2, NZ)
    pa, pb = torch.randn(ref[0].shape, generator=g), torch.randn(ref[1].shape, generator=g)
    ((ref[0] * pa.double()).sum() + (ref[1] * pb.double()).sum()).backward()
    m = m.to(cuda)
    f, c = feats.to(cuda).requires_grad_(True), fcl.to(cuda).requires_grad_(True)
    a, b, oc = m(points.to(cuda), f, coors.to(cuda), c)
    ((a * pa.to(cuda)).sum() + (b * pb.to(cuda)).sum()).backward()
    assert torch.equal(oc.cpu(), ref[2])
    errs = {"point": _rel(a, ref[0]), "group": _rel(b, ref[1]), "feats": _rel(f.grad, f_o.grad), "f_cluster": _rel(c.grad, c_o.grad)}
    errs.update({n_: _rel(p.grad, w[n_].grad) for n_, p in m.named_parameters()})
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, bad


def _check_layer(cuda, m, x, coors, fcl, want_point=True, want_group=True, fcl_grad=True, seed=0):
    """One SIRLayer (return_point_feats=True) against fp64 oracle autograd; returns the errors."""
    g = torch.Generator().manual_seed(seed)
    _, inv = torch.unique(coors, return_inverse=True, dim=0)
    G = int(inv.max()) + 1
    w = {"x." + k: v.detach().double().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    x_o = x.double().requires_grad_(True)
    c_o = fcl.double().requires_grad_(fcl_grad) if fcl is not None else None
    pf, gf = O.sir_layer_forward(x_o, inv, G, c_o, w, "x.", 3, m.num_vfe, NZ, 1e-3, m.act, 10.0, with_shortcut=m.with_shortcut)
    pp, pg = torch.randn(pf.shape, generator=g), torch.randn(gf.shape, generator=g)
    loss = (pf * pp.double()).sum() * want_point + (gf * pg.double()).sum() * want_group
    loss.backward()
    m = m.to(cuda)
    xg = x.to(cuda).requires_grad_(True)
    cg = fcl.to(cuda).requires_grad_(fcl_grad) if fcl is not None else None
    a, b = m(xg, coors.to(cuda), cg)
    terms = ([(a * pp.to(cuda)).sum()] if want_point else []) + ([(b * pg.to(cuda)).sum()] if want_group else [])
    sum(terms).backward()
    errs = {"point": _rel(a, pf), "group": _rel(b, gf), "in_feats": _rel(xg.grad, x_o.grad)}
    if fcl is not None and fcl_grad:
        errs["f_cluster"] = _rel(cg.grad, c_o.grad)
    errs.update({n_: _rel(p.grad, w["x." + n_].grad) for n_, p in m.named_parameters()})
    return errs


def _pts(N, G, cin, rel_in=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, generator=g)
    x[:, :3] *= 10
    gid = torch.randint(0, G, (N,), generator=g)
    gid[:G] = torch.arange(G)[:N]
    coors = torch.stack([torch.zeros_like(gid), gid], 1)
    return x, coors, torch.randn(N, rel_in, generator=g) * 2


def _ok(errs):
    bad = {k: v for k, v in errs.items() if not v <= TOL}
    assert not bad, bad


def test_roi_head_blocks_on_pooled_points(cuda):
    """FullySparseBboxHead's SIRLayers: in 213 then 146, rel_in 13, [128, 128], return_point_feats, many small groups."""
    x, coors, fcl = _pts(6000, 600, 213, rel_in=13, seed=1)
    _ok(_check_layer(cuda, _layer(213, [128, 128], rel_in=13, seed=2), x, coors, fcl, seed=3))
    x, coors, fcl = _pts(6000, 600, 146, rel_in=13, seed=4)
    _ok(_check_layer(cuda, _layer(146, [128, 128], rel_in=13, seed=5), x, coors, fcl, seed=6))


@pytest.mark.parametrize("case", ["f_cluster_none", "one_vfe", "relu", "shortcut", "group_only", "point_only", "f_cluster_no_grad"])
def test_sir_layer_variants(cuda, case):
    cin, feats, act = 67, [64, 64], "gelu"
    kw = dict(want_point=True, want_group=True, fcl_grad=True)
    if case == "one_vfe":
        feats = [96]
    if case == "relu":
        act = "relu"
    if case == "shortcut":
        cin = 67  # cin - 3 == C_last
    else:
        cin = 70
    if case == "group_only":
        kw["want_point"] = False
    if case == "point_only":
        kw["want_group"] = False
    if case == "f_cluster_no_grad":
        kw["fcl_grad"] = False
    x, coors, fcl = _pts(4000, 50, cin, seed=7)
    if case == "f_cluster_none":
        fcl = None
    _ok(_check_layer(cuda, _layer(cin, feats, act=act, seed=8), x, coors, fcl, seed=9, **kw))


def _composed(m):
    m._native_train = lambda: False
    return m


def test_config_scale_vs_composed(cuda):
    """150k points, 256 groups, config-3 SIR: the native path within 1e-3 of the composed torch path (both fp32) on the same GPU."""
    points, feats, coors, fcl, g = _frame(150000, 256, 79, 11)
    pa = torch.randn(150000, 128, generator=g).to(cuda)
    pb = torch.randn(256, 768, generator=g).to(cuda)
    out = []
    for native in (True, False):
        m = _sir([84, 133, 133], 128, 3).to(cuda)
        if not native:
            for blk in m.block_list:
                _composed(blk)
        f, c = feats.to(cuda).requires_grad_(True), fcl.to(cuda).requires_grad_(True)
        a, b, _ = m(points.to(cuda), f, coors.to(cuda), c)
        ((a * pa).sum() + (b * pb).sum()).backward()
        out.append(dict(point=a, group=b, feats=f.grad, f_cluster=c.grad, **{n_: p.grad for n_, p in m.named_parameters()}))
    _ok({k: _rel(out[0][k], out[1][k]) for k in out[1]})


def test_ties_go_to_the_lowest_index(cuda):
    """Rows duplicated inside a group: with a group-only gradient every later copy gets exactly 0 (the max's gradient goes to the
    lowest index), and the non-zero pattern of every gradient equals the composed path's."""
    x, coors, fcl = _pts(3000, 40, 67, seed=12)
    src = torch.arange(0, 1000, 2)
    dst = src + 1000
    x[dst], coors[dst], fcl[dst] = x[src], coors[src], fcl[src]
    grads = []
    for native in (True, False):
        m = _layer(67, [64, 64], seed=13).to(cuda)
        if not native:
            _composed(m)
        xg, cg = x.to(cuda).requires_grad_(True), fcl.to(cuda).requires_grad_(True)
        _, b = m(xg, coors.to(cuda), cg)
        (b * torch.randn(b.shape, generator=torch.Generator().manual_seed(14)).to(cuda)).sum().backward()
        grads.append([xg.grad, cg.grad] + [p.grad for p in m.parameters()])
    assert torch.all(grads[0][0][dst] == 0) and torch.all(grads[0][1][dst] == 0)
    for gn, gc in zip(grads[0], grads[1]):
        assert torch.equal(gn != 0, gc != 0)
        assert _rel(gn, gc) <= TOL


def test_backward_is_deterministic(cuda):
    points, feats, coors, fcl, g = _frame(30000, 100, 79, 15)
    m = _sir([84, 133, 133], 128, 3).to(cuda)
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        f, c = feats.to(cuda).requires_grad_(True), fcl.to(cuda).requires_grad_(True)
        a, b, _ = m(points.to(cuda), f, coors.to(cuda), c)
        (a.square().sum() + b.square().sum()).backward()
        runs.append([f.grad, c.grad] + [p.grad for p in m.parameters()])
    for x, y in zip(*runs):
        assert torch.equal(x, y)


def test_dispatch(cuda, monkeypatch):
    from sst_b200._lib import SSTB200Error
    from sst_b200.sir_modules import SIRLayer

    def boom(*a, **k):
        raise AssertionError("supported SIRLayer reached _forward_composed")

    points, feats, coors, fcl, _ = _frame(2000, 30, 79, 16)
    with monkeypatch.context() as mp:
        mp.setattr(SIRLayer, "_forward_composed", boom)
        m = _sir([84, 133, 133], 128, 3).to(cuda)
        a, b, _ = m(points.to(cuda), feats.to(cuda).requires_grad_(True), coors.to(cuda), fcl.to(cuda))
        (a.sum() + b.sum()).backward()
    # dropout > 0 trains through the composed path
    calls = []
    orig = SIRLayer._forward_composed

    def spy(self, *a, **k):
        calls.append(1)
        return orig(self, *a, **k)

    monkeypatch.setattr(SIRLayer, "_forward_composed", spy)
    x, co, fc = _pts(1000, 20, 70)
    d = _layer(70, [64, 64], dropout=0.1).to(cuda)
    pa, pb = d(x.to(cuda).requires_grad_(True), co.to(cuda), fc.to(cuda))
    (pa.sum() + pb.sum()).backward()
    assert calls
    # an out-of-range width fails in the ABI call
    bad = _layer(70, [48, 48]).to(cuda)
    with pytest.raises(SSTB200Error, match="not supported"):
        bad(x.to(cuda).requires_grad_(True), co.to(cuda), fc.to(cuda))


def test_empty_input_trains(cuda):
    m = _sir([84, 133, 133], 128, 3).to(cuda)
    f = torch.zeros(0, 79, device=cuda, requires_grad=True)
    a, b, c = m(torch.zeros(0, 5, device=cuda), f, torch.zeros(0, 3, dtype=torch.long, device=cuda), torch.zeros(0, 3, device=cuda))
    assert a.shape == (0, 128) and b.shape == (0, 768) and c.shape == (0, 3)
    (a.sum() + b.sum()).backward()
    assert f.grad.shape == (0, 79)
    assert all(p.grad is not None and not p.grad.any() for p in m.parameters())
