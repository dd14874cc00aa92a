"""GPU: FSDV2Head's native training and proposal paths (ops.cluster_head_targets with assign_xyz / code_size 10, ops.cluster_head_loss
with loss_vel, FSDV2Head.get_bboxes) against the reference's own targets (tests/golden/fsdv2_head_targets.npz) and the CPU / float64
oracle (oracle/fsdv2_head_oracle.py); VirtualVoxelFront's virtual_centroid; a small nuScenes-shaped head training a few steps.

Targets: labels, num_pos and the velocity columns and weights bit-exact, the log / sin / cos columns within one ulp.  Covered: 9- and
10-column GTs, centroid assignment with a cluster whose centre is outside a box but whose centroid is inside and the reverse, the
tasks' class order permuted against class_names.  Losses: forward and backward against float64 autograd at the bounds of
tests/test_gpu_cluster_head.py, pasted GTs (flag 0) giving no velocity loss or gradient, loss_vel over 2 * the local num_pos while
reg_avg_factor is reduced, two-run bit identity and no host sync.  get_bboxes: equal to the oracle for the Waymo `rpn` cfg and the
nuScenes test cfg with and without the all_task_max_num cut."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import cluster_head_oracle as CO
from oracle import fsdv2_head_oracle as FO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fsdv2_head_targets.npz")
LOSS_TOL = 3e-7
GRAD_TOL = 2e-6
PERM_TASKS = [['pedestrian', 'car', 'barrier', 'truck', 'bicycle'], ['bus', 'traffic_cone', 'motorcycle', 'construction_vehicle', 'trailer']]


def _dev(*a):
    return [x.to(DEV) if isinstance(x, torch.Tensor) else [y.to(DEV) for y in x] for x in a]


def _native(xyz, aux, inds, B, L, tasks=FO.NUSC_TASKS, code_size=10):
    from sst_b200 import ops
    x, a, i, Bd, Ld = _dev(xyz, aux, inds, B, L)
    return ops.cluster_head_targets(x, i, Bd, Ld, tasks, FO.NUSC_NAMES, assign_xyz=a, code_size=code_size)


def _check(got, ref):
    lab, tg, npos = got
    rl, rt, rn = ref
    assert torch.equal(npos.cpu(), rn)
    for a, b, u, v in zip(lab, rl, tg, rt):
        assert torch.equal(a.cpu(), b)
        u = u.cpu()
        assert torch.equal(u.isnan(), v.isnan())
        assert torch.equal(u[:, :3], v[:, :3]) and torch.equal(u[:, 8:], v[:, 8:])
        assert (u[:, 3:8].view(torch.int32).long() - v[:, 3:8].view(torch.int32).long()).abs().max().item() <= 1


def test_targets_match_golden_reference_and_oracle():
    g = np.load(GOLDEN)
    from oracle.make_golden_fsdv2_head import CASES
    for name in CASES:
        xyz, aux, inds = (torch.from_numpy(g[f"{name}/{k}"]) for k in ("xyz", "aux", "inds"))
        boxes, labels = torch.from_numpy(g[f"{name}/boxes"]), torch.from_numpy(g[f"{name}/labels"])
        bo = np.concatenate([[0], np.cumsum(g[f"{name}/box_sizes"])]).tolist()
        B, L = [boxes[a:b] for a, b in zip(bo, bo[1:])], [labels[a:b] for a, b in zip(bo, bo[1:])]
        lab, tg, npos = _native(xyz, aux, inds, B, L)
        for t in range(2):
            rl, rt, rw = (torch.from_numpy(g[f"{name}/{k}_t{t}"]) for k in ("labels", "targets", "weights"))
            u = tg[t].cpu()
            assert torch.equal(lab[t].cpu(), rl)
            assert torch.equal(u[:, :3], rt[:, :3]) and torch.equal(u[:, 8:10], rt[:, 8:10])
            assert (u[:, :10].view(torch.int32).long() - rt.view(torch.int32).long()).abs().max().item() <= 1
            assert torch.equal(u[:, 10], rw[:, 8])
            assert int(npos[t]) == int(((rl >= 0) & (rl < 5)).sum())
        _check((lab, tg, npos), FO.targets(xyz, inds[:, 1], B, L, FO.NUSC_TASKS, FO.NUSC_NAMES, assign_xyz=aux, code_size=10))


@pytest.mark.parametrize("width", [9, 10])
def test_targets_permuted_class_order_and_code8_centroid(width):
    xyz, aux, inds, B, L = FO.synth_clusters(20 + width, [1500, 0, 900], [40, 3, 25], width=width)
    _check(_native(xyz, aux, inds, B, L, PERM_TASKS),
           FO.targets(xyz, inds[:, 1], B, L, PERM_TASKS, FO.NUSC_NAMES, assign_xyz=aux, code_size=10))
    B7 = [b[:, :7].contiguous() for b in B]
    _check(_native(xyz, aux, inds, B7, L, PERM_TASKS, code_size=8),
           FO.targets(xyz, inds[:, 1], B7, L, PERM_TASKS, FO.NUSC_NAMES, assign_xyz=aux, code_size=8))


def test_centre_outside_centroid_inside_and_the_reverse():
    from sst_b200 import ops
    box = torch.tensor([[0.0, 0.0, -1.0, 2.0, 2.0, 2.0, 0.0, 1.5, -0.5]])           # |x|, |y| < 1, z in [-1, 1)
    xyz = torch.tensor([[1.1, 0.0, 0.0], [0.5, 0.0, 0.0]])
    aux = torch.tensor([[0.9, 0.0, 0.0], [1.3, 0.0, 0.0]])
    inds = torch.tensor([[0, 0, 0], [0, 0, 1]])
    x, a, i, b, lab = _dev(xyz, aux, inds, [box], [torch.tensor([0])])
    labels, tg, npos = ops.cluster_head_targets(x, i, b, lab, FO.NUSC_TASKS, FO.NUSC_NAMES, assign_xyz=a, code_size=10)
    assert labels[0].tolist() == [0, 5] and int(npos[0]) == 1
    t = tg[0].cpu()
    assert t[0, 0].item() == np.float32(0.0) - np.float32(1.1)                       # the encode subtracts the centre, not the centroid
    assert t[0, 8:].tolist() == [1.5, -0.5, 1.0] and t[1].abs().sum().item() == 0
    labels, _, _ = ops.cluster_head_targets(x, i, b, lab, FO.NUSC_TASKS, FO.NUSC_NAMES, code_size=10)
    assert labels[0].tolist() == [5, 0]


# ---- losses ----
def _frame(seed, width=10, n=(1500, 0, 900), m=(30, 4, 20), tasks=FO.NUSC_TASKS):
    xyz, aux, inds, B, L = FO.synth_clusters(seed, list(n), list(m), width=width)
    t = FO.targets(xyz, inds[:, 1], B, L, tasks, FO.NUSC_NAMES, assign_xyz=aux, code_size=10)
    x, r = FO.synth_preds(seed + 1, xyz.shape[0], tasks)
    return t, x, r


def _run(mode, t, x, r, reg_avg=None):
    from sst_b200 import ops
    lab, tg, npos = t
    M = x[0].shape[0]
    cfg = ops.ClusterHeadLossConfig(**FO.LOSS_MODES[mode])
    xg = [a.to(DEV).requires_grad_() for a in x]
    rg = [a.to(DEV).requires_grad_() for a in r]
    T = len(x)
    ca = torch.full((T,), float(M), device=DEV)
    ra = npos.float().to(DEV) if reg_avg is None else reg_avg.to(DEV)
    losses = ops.cluster_head_loss(xg, rg, [a.to(DEV) for a in lab], [a.to(DEV) for a in tg], npos.to(DEV), ca, ra, cfg)
    (losses * torch.linspace(0.5, 1.5, losses.numel(), device=DEV).reshape(losses.shape)).sum().backward()
    xo = [a.double().requires_grad_() for a in x]
    ro = [a.double().requires_grad_() for a in r]
    ref = FO.losses(xo, ro, lab, tg, npos, [float(M)] * T, ra.cpu().double(), **FO.LOSS_MODES[mode])
    (ref * torch.linspace(0.5, 1.5, ref.numel(), dtype=torch.float64).reshape(ref.shape)).sum().backward()
    return losses, ref, xg, rg, xo, ro


def _rel(a, b):
    if a == b:
        return 0.0
    return abs(a - b) / max(abs(b), 1e-30)


def _grel(g, ref):
    return (g.detach().cpu().double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


@pytest.mark.parametrize("mode", list(FO.LOSS_MODES))
@pytest.mark.parametrize("width", [9, 10])
def test_losses_and_gradients_match_float64(mode, width):
    t, x, r = _frame(11 + width + len(mode), width)
    losses, ref, xg, rg, xo, ro = _run(mode, t, x, r)
    assert losses.shape == (2, 5)
    errs = [_rel(a, b) for a, b in zip(losses.detach().cpu().reshape(-1).tolist(), ref.detach().reshape(-1).tolist())]
    gerrs = [_grel(a.grad, b.grad) for a, b in zip(xg + rg, xo + ro) if b.grad.abs().max() > 0]
    print(f"[fsdv2_head] {mode} width={width}: loss rel err {max(errs):.2e}, grad rel err {max(gerrs):.2e}")
    assert max(errs) < LOSS_TOL and max(gerrs) < GRAD_TOL, (errs, gerrs)


def test_pasted_gts_give_no_velocity_loss_or_gradient():
    t, x, r = _frame(41, 10)
    lab, tg, npos = t
    tg = [a.clone() for a in tg]
    pos = [(a >= 0) & (a < 5) for a in lab]
    for a, p in zip(tg, pos):
        a[p, 10] = 0.0                                      # every positive pasted
    losses, ref, xg, rg, _, _ = _run("nusc_l1", (lab, tg, npos), x, r)
    assert torch.equal(losses[:, 4].detach().cpu(), torch.zeros(2)) and (losses[:, 1:4] > 0).all()
    for g in rg:
        assert torch.count_nonzero(g.grad[:, 8:]).item() == 0
    tg[0][pos[0].nonzero()[:3, 0], 10] = 1.0                 # three genuine ones: only their rows get a velocity gradient
    _, _, _, rg, _, _ = _run("nusc_l1", (lab, tg, npos), x, r)
    assert torch.count_nonzero(rg[0].grad[:, 8:].abs().sum(1)).item() == 3


def test_loss_vel_over_local_num_pos_with_reduced_factor():
    t, x, r = _frame(5, 10, n=(800, 600), m=(20, 10))
    lab, tg, npos = t
    lab, tg = list(lab), list(tg)
    lab[1] = torch.full_like(lab[1], 5)                      # task 1: no local positive
    tg[1] = torch.zeros_like(tg[1])
    npos = npos.clone()
    npos[1] = 0
    reg_avg = npos.float() * 0.5 + 3.0                       # the all-reduced factors differ from the local counts
    losses, ref, xg, rg, xo, ro = _run("nusc_l1", (lab, tg, npos), x, r, reg_avg=reg_avg)
    assert torch.equal(losses[1, 1:].detach().cpu(), torch.zeros(4)) and torch.count_nonzero(rg[1].grad).item() == 0
    pos = (lab[0] >= 0) & (lab[0] < 5)
    want = 0.2 * ((r[0][pos][:, 8:10].double() - tg[0][pos][:, 8:10].double()).abs() * tg[0][pos][:, 10:11].double()).sum() / \
        (2 * int(npos[0]))
    assert _rel(float(losses[0, 4]), float(want)) < LOSS_TOL
    assert max(_rel(a, b) for a, b in zip(losses.detach().cpu().reshape(-1).tolist(), ref.detach().reshape(-1).tolist())) < LOSS_TOL


def test_two_runs_are_bit_identical():
    t, x, r = _frame(31, 10, n=(20000, 15000), m=(80, 60))
    outs = []
    for _ in range(2):
        losses, _, xg, rg, _, _ = _run("nusc_smoothl1", t, x, r)
        outs.append([losses.detach()] + [a.grad for a in xg + rg])
    for a, b in zip(*outs):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def _nusc_head(**kw):
    from sst_b200.registry import MODELS
    return MODELS.build(dict(FO.NUSC_HEAD, **kw))


def test_loss_keys_and_no_host_sync():
    head = _nusc_head(in_channel=32, shared_mlp_dims=[64], train_cfg=FO.NUSC_TRAIN_CFG).to(DEV).train()
    xyz, aux, inds, B, L = FO.synth_clusters(3, [3000, 2000], [30, 20], width=10)
    xyz, aux, inds, B, L = _dev(xyz, aux, inds, B, L)
    feats = torch.randn(xyz.shape[0], 32, device=DEV)
    for check in (False, True):       # the first call grows the context arena (a cudaMalloc, which sync debug mode does not see)
        torch.cuda.synchronize()
        if check:
            torch.cuda.set_sync_debug_mode("error")
        try:
            out = head(feats)
            losses = head.loss(out['cls_logits'], out['reg_preds'], xyz, inds, B, L, aux_xyz=aux)
            sum(losses.values()).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    keys = ("loss_cls", "loss_center", "loss_size", "loss_rot", "loss_vel")
    assert list(losses) == [f"{k}.task{t}" for t in range(2) for k in keys]
    assert all(head.print_info[f"n_pos_t{t}"].is_cuda and head.print_info[f"n_pos_t{t}"].shape == (1,) for t in range(2))
    with pytest.raises(ValueError):
        head.loss(out['cls_logits'], out['reg_preds'], xyz, inds, B, L)      # centroid_assign without aux_xyz


# ---- get_bboxes ----
def _distinct_logits(M, tasks, seed):
    n = M * sum(len(t) for t in tasks)
    p = torch.linspace(0.02, 0.98, n)[torch.randperm(n, generator=torch.Generator().manual_seed(seed))]
    return [torch.logit(q).reshape(M, len(t)) for q, t in zip(p.split([M * len(t) for t in tasks]), tasks)]


@pytest.mark.parametrize("case", ["waymo_rpn", "nusc_test", "nusc_test_topk", "nusc_permuted"])
def test_get_bboxes_match_oracle(case):
    from sst_b200.registry import MODELS
    if case == "waymo_rpn":
        names, tasks, code = CO.WAYMO_NAMES, CO.WAYMO_TASKS, 8
        head = MODELS.build(dict(FO.WAYMO_HEAD, in_channel=8, shared_mlp_dims=[8], train_cfg=FO.WAYMO_TRAIN_CFG)).train()
        cfg, topk = FO.WAYMO_RPN_CFG, None
    else:
        names, tasks, code = FO.NUSC_NAMES, PERM_TASKS if case == "nusc_permuted" else FO.NUSC_TASKS, 10
        topk = 150 if case == "nusc_test_topk" else 500
        cfg = dict(FO.NUSC_TEST_CFG, all_task_max_num=topk)
        head = _nusc_head(in_channel=8, shared_mlp_dims=[8], tasks=[dict(class_names=t) for t in tasks], test_cfg=cfg).eval()
    xyz, _, inds, _, _ = FO.synth_clusters(9, [700, 300, 0], [40, 20, 0], names, spread=15.0)
    M = xyz.shape[0]
    _, r = FO.synth_preds(4, M, tasks, code)
    r = [v * 0.3 for v in r]
    x = _distinct_logits(M, tasks, 4)
    x, r, xyz, inds = [a.to(DEV) for a in x], [a.to(DEV) for a in r], xyz.to(DEV), inds.to(DEV)
    got = head.get_bboxes(x, r, xyz, inds, [dict()] * 3)
    ref = FO.get_bboxes(x, r, xyz, inds[:, 1], 3, tasks, names, cfg, topk)
    for (a, s, lab), (ra, rs, rl) in zip(got, ref):
        assert torch.equal(a.cpu(), ra) and torch.equal(s.cpu(), rs) and torch.equal(lab.cpu(), rl)
    assert got[0][0].shape[1] == (9 if code == 10 else 7)
    if case == "nusc_test_topk":
        assert got[0][0].shape[0] == topk and FO.get_bboxes(x, r, xyz, inds[:, 1], 3, tasks, names, cfg)[0][0].shape[0] > topk


def test_get_bboxes_topk_adds_no_host_sync(monkeypatch):
    """the all_task_max_num cut adds no host sync to the NMS's two"""
    head = _nusc_head(in_channel=8, shared_mlp_dims=[8], test_cfg=dict(FO.NUSC_TEST_CFG, all_task_max_num=50)).eval()
    xyz, _, inds, _, _ = FO.synth_clusters(2, [800, 700], [20, 20], spread=15.0)
    x, r = FO.synth_preds(2, xyz.shape[0], FO.NUSC_TASKS)
    args = ([a.to(DEV) for a in x], [a.to(DEV) for a in r], xyz.to(DEV), inds.to(DEV), [dict()] * 2)
    head.get_bboxes(*args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    import warnings
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out = head.get_bboxes(*args)
    torch.cuda.set_sync_debug_mode("default")
    assert len([m for m in w if "synchroniz" in str(m.message)]) == 2
    assert all(o[0].shape[0] == 50 for o in out)


# ---- virtual_centroid ----
def test_virtual_centroid_is_the_per_voxel_mean():
    from sst_b200.fsdv2_modules import VirtualVoxelFront
    g = torch.Generator().manual_seed(0)
    vs, rng = [0.4, 0.4, 0.4], [-20.0, -20.0, -4.0, 20.0, 20.0, 4.0]
    norm = dict(type='naiveSyncBN1d', eps=1e-3, momentum=0.01)
    m = VirtualVoxelFront(
        voxel_encoder=dict(type='DynamicScatterVFE', in_channels=19, feat_channels=[32, 32], with_cluster_center=True,
                           with_voxel_center=True, voxel_size=vs, point_cloud_range=rng, norm_cfg=norm, unique_once=True,
                           rel_dist_scaler=10.0),
        virtual_point_projector=dict(in_channels=24, hidden_dims=[16, 16], norm_cfg=norm, ori_in_channels=19, ori_hidden_dims=[16, 16]),
        train_cfg=dict(centroid_assign=True)).to(DEV)
    n_o, n_s = 6000, 3000
    ori = torch.cat([(torch.rand(n_o, 3, generator=g) - 0.5) * torch.tensor([30.0, 30.0, 6.0]), torch.rand(n_o, 2, generator=g)], 1)
    smp = torch.cat([ori[:n_s, :3] + torch.randn(n_s, 3, generator=g) * 0.2, torch.rand(n_s, 2, generator=g)], 1)
    sampled = dict(seg_points=smp, center_preds=smp[:, :3] + torch.randn(n_s, 3, generator=g) * 0.3, seg_logits=torch.randn(n_s, 3),
                   seg_feats=torch.randn(n_s, 16, generator=g), batch_idx=torch.randint(0, 2, (n_s,), generator=g))
    origin = dict(seg_points=ori, seg_feats=torch.randn(n_o, 19, generator=g), batch_idx=torch.randint(0, 2, (n_o,), generator=g))
    sampled, origin = ({k: v.to(DEV) for k, v in d.items()} for d in (sampled, origin))
    for training in (True, False):
        m.train(training)
        with torch.no_grad():
            fr = m.front(sampled, origin)
            out = m.finish(fr, fr["voxel_feats"], fr["voxel_coors"])
        assert ("virtual_centroid" in out) == training
    inv, pts, vm = fr["unq_inv"].cpu(), fr["cat_pts"][:, :3].cpu().double(), fr["virtual_mask"].cpu()
    n = fr["voxel_coors"].shape[0]
    ref = torch.zeros(n, 3, dtype=torch.float64).index_add_(0, inv, pts) / torch.bincount(inv, minlength=n)[:, None].double()
    m.train(True)
    with torch.no_grad():
        out = m.finish(fr, fr["voxel_feats"], fr["voxel_coors"])
    got = out["virtual_centroid"].cpu().double()
    assert got.shape == (int(vm.sum()), 3) and (got - ref[vm]).abs().max().item() < 1e-5
    half = torch.tensor(vs, dtype=torch.float64) / 2 + 1e-3
    assert ((got - out["virtual_centers"].cpu().double()).abs() < half).all()
    with pytest.raises(ValueError):
        VirtualVoxelFront(voxel_encoder=dict(type='DynamicScatterVFE', in_channels=19, feat_channels=[32], voxel_size=vs,
                                             point_cloud_range=rng, norm_cfg=norm),
                          virtual_point_projector=dict(in_channels=24, hidden_dims=[16], norm_cfg=norm, ori_in_channels=19,
                                                       ori_hidden_dims=[16]), train_cfg=dict(centroid_alpha=0.5))


# ---- training ----
def test_nusc_head_trains():
    """A few Adam steps of a small nuScenes-shaped FSDV2Head (naiveSyncBN1d, two 5-class tasks, code size 10, centroid assignment)
    on fixed features of synthetic clusters: the summed loss falls and every parameter gets a finite gradient."""
    torch.manual_seed(0)
    head = _nusc_head(in_channel=32, shared_mlp_dims=[64, 64], train_cfg=FO.NUSC_TRAIN_CFG,
                      common_attrs=dict(center=(3, 2, 32), dim=(3, 2, 32), rot=(2, 2, 32), vel=(2, 2, 32)), cls_hidden_dim=32).to(DEV).train()
    xyz, aux, inds, B, L = FO.synth_clusters(3, [600, 500], [40, 30], width=10, inside=0.8)
    g = torch.Generator().manual_seed(1)
    feats = torch.cat([xyz / 30.0, torch.randn(xyz.shape[0], 29, generator=g)], 1)
    xyz, aux, inds, B, L, feats = _dev(xyz, aux, inds, B, L, feats)
    opt = torch.optim.Adam(head.parameters(), lr=2e-3)
    totals = []
    for step in range(8):
        opt.zero_grad()
        out = head(feats)
        losses = head.loss(out['cls_logits'], out['reg_preds'], xyz, inds, B, L, aux_xyz=aux)
        loss = sum(losses.values())
        loss.backward()
        totals.append(loss.item())
        for n_, p in head.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), (step, n_)
        opt.step()
    print(f"[fsdv2_head] nuScenes head losses {['%.4f' % v for v in totals]}")
    assert all(math.isfinite(v) for v in totals) and totals[-1] < totals[0]
