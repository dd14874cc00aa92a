"""GPU: SparseClusterHeadV2's native training and proposal paths (ops.cluster_head_targets, ops.cluster_head_loss,
ops.multiclass_nms_groups) against the reference's own targets (tests/golden/cluster_head_targets.npz) and the CPU / float64 oracle
(oracle/cluster_head_oracle.py), the module built from the D1 config, and a D1 SIR + head training a few steps.

Targets: labels and num_pos bit-exact; bbox targets exact in the delta columns and within one ulp of the rounded float64 values in the
log / sin / cos columns (the oracle rounds them once from float64; the kernel's double log / sin / cos are within an ulp of correctly
rounded).  Covered: B = 1, 2, 3, 8 with samples without clusters or GTs, clusters not sorted by sample, Argoverse 2's six multi-class
groups with boxes stacked across classes, negative-label and no-task GTs, G = 255, 256, 257 (the 256-GT shared-memory chunk) and the
4096 cap, 4097 refused, clusters on box faces and one ulp either side, yaws of +-pi, an out-of-range batch index, outputs pre-filled
with NaN / 0xFF through the C ABI.

Losses: forward and backward against float64 autograd with focal gamma 2 / alpha 0.25 and gamma 1, L1 and SmoothL1 (beta 0.1), logits
out to +-40, a task without positives, the local-zero / reduced-positive factor, NaN logits, two-run bit identity and no host sync.
Bounds are VoteSeg's (relative to the float64 value; gradients elementwise relative to the largest gradient); the worst seen on an
H100 80GB HBM3 was 7.2e-8 on the losses and 3.7e-7 on the gradients.

get_bboxes: equal to the oracle's per-(task, sample) box3d_multiclass_nms for the training `rpn` cfg and the test cfg, with a
(sample, task) group over max_num and a batch of one with out-of-range batch indices; one host sync per call for the `rpn` cfg, two
with NMS.  Misuse: off-device loss inputs raise; strided targets are read correctly."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import cluster_head_oracle as CO
from oracle import voteseg_oracle as VO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "cluster_head_targets.npz")
LOSS_TOL = 3e-7       # relative; worst seen 7.2e-8
GRAD_TOL = 2e-6       # max |err| / max |grad|; worst seen 3.7e-7


def _native_targets(xyz, inds, B, L, tasks, names):
    from sst_b200 import ops
    return ops.cluster_head_targets(xyz.to(DEV), inds.to(DEV), [b.to(DEV) for b in B], [lab.to(DEV) for lab in L], tasks, names)


def _check_targets(got, ref):
    lab, tg, npos = got
    rl, rt, rn = ref
    assert torch.equal(npos.cpu(), rn)
    for a, b, u, v in zip(lab, rl, tg, rt):
        assert torch.equal(a.cpu(), b)
        u = u.cpu()
        assert torch.equal(u.isnan(), v.isnan())
        ok = ~v.isnan().any(1)
        assert torch.equal(u[ok][:, :3], v[ok][:, :3])
        ulp = (u[ok][:, 3:].view(torch.int32).long() - v[ok][:, 3:].view(torch.int32).long()).abs()
        assert ulp.numel() == 0 or ulp.max().item() <= 1


def _oracle_targets(xyz, inds, B, L, tasks, names):
    return CO.targets(xyz, inds[:, 1], B, L, tasks, names)


# ---- targets ----
def test_targets_match_golden_reference():
    g = np.load(GOLDEN)
    from oracle.make_golden_cluster_head import CASES
    for name, (names, tasks, _, _) in CASES.items():
        xyz, inds = torch.from_numpy(g[f"{name}/xyz"]), torch.from_numpy(g[f"{name}/inds"])
        boxes, labels = torch.from_numpy(g[f"{name}/boxes"]), torch.from_numpy(g[f"{name}/labels"])
        bo = np.concatenate([[0], np.cumsum(g[f"{name}/box_sizes"])]).tolist()
        B = [boxes[a:b] for a, b in zip(bo, bo[1:])]
        L = [labels[a:b] for a, b in zip(bo, bo[1:])]
        lab, tg, npos = _native_targets(xyz, inds, B, L, tasks, names)
        for t in range(len(tasks)):
            rl, rt = torch.from_numpy(g[f"{name}/labels_t{t}"]), torch.from_numpy(g[f"{name}/targets_t{t}"])
            assert torch.equal(lab[t].cpu(), rl)
            u = tg[t].cpu()
            assert torch.equal(u[:, :3], rt[:, :3])
            assert (u.view(torch.int32).long() - rt.view(torch.int32).long()).abs().max().item() <= 1
            assert int(npos[t]) == int(((rl >= 0) & (rl < len(tasks[t]))).sum())
        _check_targets((lab, tg, npos), _oracle_targets(xyz, inds, B, L, tasks, names))


@pytest.mark.parametrize("sizes", [([900], [20]), ([0, 700], [5, 12]), ([1200, 300, 0], [30, 0, 7]),
                                   ([500, 0, 800, 300, 0, 1000, 20, 400], [10, 3, 0, 25, 0, 40, 2, 9])], ids=["B1", "B2", "B3", "B8"])
@pytest.mark.parametrize("case", ["waymo", "argo"])
def test_targets_match_oracle(sizes, case):
    names, tasks = (CO.WAYMO_NAMES, CO.WAYMO_TASKS) if case == "waymo" else (CO.ARGO_NAMES, CO.ARGO_TASKS)
    n, m = sizes
    xyz, inds, B, L = CO.synth_clusters(len(n) * 17 + len(names), n, m, names, invalid=0.1)
    for b in range(len(B)):
        if B[b].shape[0] > 1:
            B[b][1::2] = B[b][0:-1:2]                      # boxes of two classes stacked: the rank order decides
            CO.yaw_pi(B[b])
        if n[b] and m[b] >= 3:
            xyz = torch.cat([xyz, VO.face_points(B[b][:3])])
            inds = torch.cat([inds, torch.tensor([[0, b, 0]]).repeat(xyz.shape[0] - inds.shape[0], 1)])
    if case == "waymo" and sum(m):
        L[int(np.argmax(m))][0] = 7                        # a class in no task
    _check_targets(_native_targets(xyz, inds, B, L, tasks, names), _oracle_targets(xyz, inds, B, L, tasks, names))


@pytest.mark.parametrize("G", [1, 255, 256, 257, 4096])
def test_targets_gt_chunk_edges(G):
    g = torch.Generator().manual_seed(G)
    boxes, _ = VO.synth_boxes(g, G, 3, spread=30.0)
    lab = torch.randint(0, 3, (G,), generator=g)
    pts = torch.cat([VO.points_around(g, boxes, 3000, spread=30.0, cols=3), VO.points_around(g, boxes[-3:], 60, 30.0, cols=3, inside=1.0)])
    inds = torch.stack([torch.zeros(pts.shape[0], dtype=torch.long), (torch.arange(pts.shape[0]) % 2), torch.arange(pts.shape[0])], 1)
    B, L = [boxes, boxes[:G // 2]], [lab, lab[:G // 2]]
    _check_targets(_native_targets(pts, inds, B, L, CO.WAYMO_TASKS, CO.WAYMO_NAMES),
                   _oracle_targets(pts, inds, B, L, CO.WAYMO_TASKS, CO.WAYMO_NAMES))


def test_targets_refuse_more_than_the_gt_cap():
    from sst_b200 import _lib
    g = torch.Generator().manual_seed(1)
    boxes, _ = VO.synth_boxes(g, 4097, 3)
    with pytest.raises(_lib.SSTB200Error, match="at most 4096"):
        _native_targets(torch.zeros(10, 3), torch.zeros(10, 3, dtype=torch.long), [boxes], [torch.zeros(4097, dtype=torch.long)],
                        CO.WAYMO_TASKS, CO.WAYMO_NAMES)


def test_out_of_range_batch_index_and_dirty_outputs_through_c_abi():
    from sst_b200 import _lib as L_
    xyz, inds, B, L = CO.synth_clusters(5, [700, 500], [20, 15], CO.WAYMO_NAMES)
    inds[3, 1], inds[10, 1] = 2, -1                          # outside [0, B)
    ref = _oracle_targets(xyz, inds, B, L, CO.WAYMO_TASKS, CO.WAYMO_NAMES)
    assert all(int(r[3]) == -1 and int(r[10]) == -1 for r in ref[0])
    M = xyz.shape[0]
    labels = [torch.full((M,), -7, dtype=torch.int64, device=DEV) for _ in range(3)]
    tg = [torch.full((M, 8), float("nan"), device=DEV) for _ in range(3)]
    npos = torch.full((3,), -1, dtype=torch.int64, device=DEV)
    x, i_ = xyz.to(DEV), inds.to(DEV)
    gt, gl = torch.cat(B).to(DEV), torch.cat(L).to(DEV)
    c = L_.ctx(DEV)
    P = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])  # noqa: E731
    L_.check(c, L_.lib().sstb200_cluster_head_targets(c, x.data_ptr(), 3, i_.data_ptr() + 8, 3, M, gt.data_ptr(), gl.data_ptr(),
                                                      L_.arr(C.c_int32, [0, 20, 35]), 2, 3, L_.arr(C.c_int32, [0, 1, 2]),
                                                      L_.arr(C.c_int32, [0, 0, 0]), 3, L_.arr(C.c_int32, [1, 1, 1]), P(labels), P(tg),
                                                      npos.data_ptr()))
    _check_targets((labels, tg, npos), ref)
    # the loss of such a cluster is NaN
    from sst_b200 import ops
    xs, rs = CO.synth_preds(1, M, CO.WAYMO_TASKS)
    losses = ops.cluster_head_loss([a.to(DEV) for a in xs], [a.to(DEV) for a in rs], labels, tg, npos,
                                   torch.full((3,), float(M), device=DEV), npos.float(), ops.ClusterHeadLossConfig(**CO.LOSS_MODES["fsd_l1"]))
    assert losses[:, 0].isnan().all() and not losses[:, 1:].isnan().any()


# ---- losses ----
def _frame(seed, mode, n=(1500, 0, 900), m=(30, 4, 0), wide=False, case="waymo"):
    names, tasks = (CO.WAYMO_NAMES, CO.WAYMO_TASKS) if case == "waymo" else (CO.ARGO_NAMES, CO.ARGO_TASKS)
    xyz, inds, B, L = CO.synth_clusters(seed, list(n), list(m), names)
    t = _oracle_targets(xyz, inds, B, L, tasks, names)
    x, r = CO.synth_preds(seed, xyz.shape[0], tasks, scale=4.0)
    if wide:
        for a in x:
            a[::13] = 40.0 * torch.sign(torch.randn(a[::13].shape, generator=torch.Generator().manual_seed(seed)))
    return t, x, r


def _run(mode, t, x, r, cls_avg=None, reg_avg=None):
    from sst_b200 import ops
    lab, tg, npos = t
    M = x[0].shape[0]
    xg = [a.to(DEV).requires_grad_(True) for a in x]
    rg = [a.to(DEV).requires_grad_(True) for a in r]
    ca = torch.full((len(x),), float(M), device=DEV) if cls_avg is None else cls_avg.to(DEV)
    ra = npos.float().to(DEV) if reg_avg is None else reg_avg.to(DEV)
    losses = ops.cluster_head_loss(xg, rg, [a.to(DEV) for a in lab], [a.to(DEV) for a in tg], npos.to(DEV), ca, ra,
                                   ops.ClusterHeadLossConfig(**CO.LOSS_MODES[mode]))
    xo, ro = [a.double().requires_grad_(True) for a in x], [a.double().requires_grad_(True) for a in r]
    ref = CO.losses(xo, ro, lab, tg, npos, ca.cpu().double(), ra.cpu().double(), **CO.LOSS_MODES[mode])
    w = torch.linspace(0.5, 1.5, losses.numel()).reshape(losses.shape)
    (losses * w.to(DEV)).sum().backward()
    (ref * w.double()).sum().backward()
    return losses, ref, xg, rg, xo, ro


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-30)


def _grel(g, ref):
    return (g.detach().cpu().double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


@pytest.mark.parametrize("mode", list(CO.LOSS_MODES))
@pytest.mark.parametrize("wide", [False, True], ids=["randn", "pm40"])
def test_losses_and_gradients_match_float64(mode, wide):
    t, x, r = _frame(11 + sum(map(ord, mode)), mode, wide=wide, case="argo" if mode.startswith("argo") else "waymo")
    losses, ref, xg, rg, xo, ro = _run(mode, t, x, r)
    errs = [_rel(a, b) for a, b in zip(losses.detach().cpu().reshape(-1).tolist(), ref.detach().reshape(-1).tolist())]
    gerrs = [_grel(a.grad, b.grad) for a, b in zip(xg + rg, xo + ro) if b.grad.abs().max() > 0]
    print(f"[cluster_head] {mode} wide={wide}: loss rel err {max(errs):.2e}, grad rel err {max(gerrs):.2e}")
    assert max(errs) < LOSS_TOL and max(gerrs) < GRAD_TOL, (errs, gerrs)


def test_task_without_positives_and_reduced_factor():
    t, x, r = _frame(5, "fsd_l1", n=(800, 600), m=(20, 10))
    lab, tg, npos = t
    lab[1] = torch.full_like(lab[1], 1)                     # task 1: no local positive
    tg[1] = torch.zeros_like(tg[1])
    npos = npos.clone()
    npos[1] = 0
    reg_avg = npos.float()
    reg_avg[1] = 3.0                                        # the all-reduced factor is positive
    losses, ref, xg, rg, xo, ro = _run("fsd_l1", (lab, tg, npos), x, r, reg_avg=reg_avg)
    assert torch.equal(losses[1, 1:].detach().cpu(), torch.zeros(3))
    assert torch.count_nonzero(rg[1].grad).item() == 0
    assert max(_rel(a, b) for a, b in zip(losses.detach().cpu().reshape(-1).tolist(), ref.detach().reshape(-1).tolist())) < LOSS_TOL


def test_nan_logit_poisons_only_its_own_gradient():
    t, x, r = _frame(21, "fsd_l1")
    x = [a.clone() for a in x]
    x[0][7, 0] = float("nan")
    losses, _, xg, rg, _, _ = _run("fsd_l1", t, x, r)
    assert math.isnan(losses[0, 0].item()) and not losses[1:, 0].isnan().any() and not losses[:, 1:].isnan().any()
    g = xg[0].grad.cpu()
    assert g[7, 0].isnan() and g.isnan().sum().item() == 1 and not any(a.grad.isnan().any() for a in xg[1:] + rg)


def test_two_runs_are_bit_identical():
    t, x, r = _frame(31, "argo_smoothl1", n=(20000, 15000), m=(80, 60), case="argo")
    outs = []
    for _ in range(2):
        losses, _, xg, rg, _, _ = _run("argo_smoothl1", t, x, r)
        outs.append([losses.detach()] + [a.grad for a in xg + rg])
    for a, b in zip(*outs):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_no_host_sync():
    from sst_b200.registry import MODELS
    head = MODELS.build(dict(CO.FSD_D1_HEAD, in_channel=32, shared_mlp_dims=[64], train_cfg=CO.FSD_D1_TRAIN_CFG)).to(DEV).train()
    xyz, inds, B, L = CO.synth_clusters(3, [3000, 2000], [30, 20], CO.WAYMO_NAMES)
    xyz, inds, B, L = xyz.to(DEV), inds.to(DEV), [b.to(DEV) for b in B], [lab.to(DEV) for lab in L]
    feats = torch.randn(xyz.shape[0], 32, device=DEV)
    for check in (False, True):       # the first call grows the context arena (a cudaMalloc, which sync debug mode does not see)
        torch.cuda.synchronize()
        if check:
            torch.cuda.set_sync_debug_mode("error")
        try:
            out = head(feats)
            losses = head.loss(out['cls_logits'], out['reg_preds'], xyz, inds, B, L)
            sum(losses.values()).backward()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert list(losses) == [f"{k}.task{t}" for t in range(3) for k in ("loss_cls", "loss_center", "loss_size", "loss_rot")]


# ---- get_bboxes ----
@pytest.mark.parametrize("cfg", ["rpn", "test"])
@pytest.mark.parametrize("case", ["waymo", "argo"])
def test_get_bboxes_match_oracle(cfg, case):
    from sst_b200.registry import MODELS
    names, tasks = (CO.WAYMO_NAMES, CO.WAYMO_TASKS) if case == "waymo" else (CO.ARGO_NAMES, CO.ARGO_TASKS)
    head = MODELS.build(dict(CO.FSD_D1_HEAD, num_classes=len(names), class_names=names, tasks=[dict(class_names=t) for t in tasks],
                             in_channel=8, shared_mlp_dims=[8], train_cfg=CO.FSD_D1_TRAIN_CFG, test_cfg=CO.FSD_D1_TEST_CFG))
    head.train(cfg == "rpn")
    # sample 0 puts more than max_num = 500 boxes above the score threshold in one (sample, task) group
    xyz, inds, B, L = CO.synth_clusters(9, [1400, 300, 0], [40, 20, 0], names, spread=15.0)
    M = xyz.shape[0]
    _, r = CO.synth_preds(4, M, tasks)
    r = [v * 0.3 for v in r]
    # distinct scores: the max_num cut is the reference's unstable descending sort, whose order of tied scores is the sort's own
    n = [M * len(t) for t in tasks]
    p = torch.linspace(0.02, 0.98, sum(n))[torch.randperm(sum(n), generator=torch.Generator().manual_seed(4))]
    x = [torch.logit(q).reshape(M, len(t)) for q, t in zip(p.split(n), tasks)]
    inds[5, 1] = 7                                           # outside [0, B): dropped, as the reference's split drops it
    x, r, xyz, inds = [a.to(DEV) for a in x], [a.to(DEV) for a in r], xyz.to(DEV), inds.to(DEV)
    got = head.get_bboxes(x, r, xyz, inds, [dict()] * 3)
    # the oracle's per-(task, sample) composition on the same device: its decode and sigmoid are the reference's GPU ops
    ref = CO.get_bboxes(x, r, xyz, inds[:, 1], 3, tasks, names, CO.RPN_CFG if cfg == "rpn" else CO.TEST_CFG)
    for (a, s, l), (ra, rs, rl) in zip(got, ref):
        assert torch.equal(a.cpu(), ra) and torch.equal(s.cpu(), rs) and torch.equal(l.cpu(), rl)
    assert ref[0][0].shape[0] >= 500
    assert torch.cat([a.sigmoid().reshape(-1) for a in x]).cpu().unique().numel() == sum(n)


@pytest.mark.parametrize("cfg", ["rpn", "test"])
def test_get_bboxes_host_syncs(monkeypatch, cfg):
    """whatever B and T: one host sync per call for the training `rpn` cfg (no NMS: every candidate is kept), two with NMS (the
    candidate counts, then the kept counts)"""
    from sst_b200.registry import MODELS
    head = MODELS.build(dict(CO.FSD_D1_HEAD, in_channel=8, shared_mlp_dims=[8], train_cfg=CO.FSD_D1_TRAIN_CFG,
                             test_cfg=CO.FSD_D1_TEST_CFG)).train(cfg == "rpn")
    xyz, inds, _, _ = CO.synth_clusters(2, [800, 700, 600, 500], [10] * 4, CO.WAYMO_NAMES)
    x, r = CO.synth_preds(2, xyz.shape[0], CO.WAYMO_TASKS)
    args = ([a.to(DEV) for a in x], [a.to(DEV) for a in r], xyz.to(DEV), inds.to(DEV), [dict()] * 4)
    head.get_bboxes(*args)
    calls = []
    real = torch.Tensor.tolist
    monkeypatch.setattr(torch.Tensor, "tolist", lambda self: (calls.append(self.is_cuda), real(self))[1])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    import warnings
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        head.get_bboxes(*args)
    torch.cuda.set_sync_debug_mode("default")
    syncs = [m for m in w if "synchroniz" in str(m.message)]
    want = 1 if cfg == "rpn" else 2
    assert calls == [True] * want and len(syncs) == want, (calls, [str(m.message) for m in syncs])


def test_get_bboxes_batch_of_one_keeps_every_cluster():
    """B = 1: every cluster belongs to the sample, out-of-range batch index or not, as the reference's split_by_batch gives it"""
    from sst_b200.registry import MODELS
    head = MODELS.build(dict(CO.FSD_D1_HEAD, in_channel=8, shared_mlp_dims=[8], train_cfg=CO.FSD_D1_TRAIN_CFG,
                             test_cfg=CO.FSD_D1_TEST_CFG)).eval()
    xyz, inds, _, _ = CO.synth_clusters(5, [400], [20], CO.WAYMO_NAMES, spread=15.0)
    inds[3, 1], inds[9, 1] = 4, -1
    x, r = CO.synth_preds(6, xyz.shape[0], CO.WAYMO_TASKS)
    x, r, xyz, inds = [a.to(DEV) for a in x], [a.to(DEV) for a in r], xyz.to(DEV), inds.to(DEV)
    (a, s, l), = head.get_bboxes(x, r, xyz, inds, [dict()])
    (ra, rs, rl), = CO.get_bboxes(x, r, xyz, inds[:, 1], 1, CO.WAYMO_TASKS, CO.WAYMO_NAMES, CO.TEST_CFG)
    assert torch.equal(a.cpu(), ra) and torch.equal(s.cpu(), rs) and torch.equal(l.cpu(), rl)


def test_loss_refuses_off_device_inputs_and_reads_strided_targets():
    """a host or wrong-device input raises before any kernel; a strided bbox_targets view gives the contiguous result"""
    from sst_b200 import _lib, ops
    t, x, r = _frame(8, "fsd_l1")
    lab, tg, npos = t
    M = x[0].shape[0]
    cfg = ops.ClusterHeadLossConfig(**CO.LOSS_MODES["fsd_l1"])
    xg, rg = [a.to(DEV) for a in x], [a.to(DEV) for a in r]
    ld, td, nd = [a.to(DEV) for a in lab], [a.to(DEV) for a in tg], npos.to(DEV)
    ca, ra = torch.full((3,), float(M), device=DEV), nd.float()
    for kw in (dict(num_pos=npos), dict(labels=[lab[0]] + ld[1:]), dict(bbox_targets=td[:2] + [tg[2]]),
               dict(cls_avg_factor=ca.cpu()), dict(reg_avg_factor=ra.cpu())):
        a = dict(cls_logits=xg, reg_preds=rg, labels=ld, bbox_targets=td, num_pos=nd, cls_avg_factor=ca, reg_avg_factor=ra)
        a.update(kw)
        with pytest.raises(_lib.SSTB200Error, match="CUDA tensor on"):
            ops.cluster_head_loss(**a, cfg=cfg)
    wide = [torch.cat([a, torch.full_like(a, float("nan"))], 1)[:, :8] for a in td]      # row stride 16
    assert not wide[0].is_contiguous()
    got = ops.cluster_head_loss(xg, rg, ld, wide, nd, ca, ra, cfg)
    ref = ops.cluster_head_loss(xg, rg, ld, td, nd, ca, ra, cfg)
    assert torch.equal(got, ref)


# ---- module ----
def test_head_forward_matches_float64_and_refusals():
    from sst_b200.registry import MODELS
    from sst_b200.cluster_head_modules import SparseClusterHeadV2
    torch.manual_seed(0)
    head = MODELS.build(dict(CO.FSD_D1_HEAD, train_cfg=CO.FSD_D1_TRAIN_CFG, test_cfg=CO.FSD_D1_TEST_CFG))
    ref = MODELS.build(dict(CO.FSD_D1_HEAD))
    ref.load_state_dict(head.state_dict())
    ref = ref.double().eval()
    head = head.to(DEV).eval()
    feats = torch.randn(2000, 768, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        a, b = head(feats.to(DEV)), ref(feats.double())
    for k in ("cls_logits", "reg_preds"):
        for u, v in zip(a[k], b[k]):
            assert _grel(u, v) < 1e-4, k
    assert head.sync_reg_avg_factor and not head.sync_cls_avg_factor
    base = dict(CO.FSD_D1_HEAD)
    base.pop("type")
    for kw in (dict(loss_iou=dict(type="CrossEntropyLoss")), dict(iou_mlp=[64]), dict(corner_loss_cfg=dict(delta=1.0)),
               dict(enlarge_width=0.1), dict(loss_vel=dict(type="L1Loss")), dict(bbox_coder=dict(type="BasePointBBoxCoder", code_size=10)),
               dict(loss_cls=dict(type="CrossEntropyLoss")), dict(loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=0.5)),
               dict(loss_center=dict(type="L1Loss", reduction="sum")), dict(loss_size=dict(type="SmoothL1Loss", beta=0.1)),
               dict(loss_rot=dict(type="GIoULoss"))):
        with pytest.raises(ValueError):
            SparseClusterHeadV2(**dict(base, **kw))
    h = SparseClusterHeadV2(**base)
    for cfg in (dict(assign_by_dist=True), dict(max_assign_dist=2.0), dict(code_weight=[1.0] * 8)):
        with pytest.raises(ValueError):
            h.train_cfg = cfg


# ---- training ----
def test_d1_sir_and_head_train():
    """A few Adam steps of a D1-shaped SIR cluster backbone (3 blocks, [128, 128], GELU) and the D1 SparseClusterHeadV2 on synthetic
    clustered Waymo-shaped points with GTs: the summed loss falls and every SIR and head parameter gets a finite, non-zero gradient."""
    from sst_b200.registry import MODELS
    from sst_b200.sir_modules import SIR
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(3)
    Bn, G_per = 2, 300
    xyz_c, inds, Bx, L = CO.synth_clusters(3, [G_per] * Bn, [40] * Bn, CO.WAYMO_NAMES, spread=40.0, shuffle=False, inside=0.7)
    G = xyz_c.shape[0]
    gid = torch.arange(G).repeat_interleave(20)
    pts = xyz_c[gid] + torch.randn(gid.shape[0], 3, generator=g) * 0.3
    points = torch.cat([pts, torch.rand(gid.shape[0], 2, generator=g)], 1)
    coors = torch.stack([inds[gid, 0], inds[gid, 1], gid], 1)
    feats = torch.randn(gid.shape[0], 79, generator=g)
    fcl = (pts - xyz_c[gid])
    sir = SIR(num_blocks=3, in_channels=[84, 133, 133], feat_channels=[[128, 128]] * 3, rel_mlp_hidden_dims=[[16, 32]] * 3,
              norm_cfg=dict(type='LN', eps=1e-3), mode='max', xyz_normalizer=[20, 20, 4], act='gelu', unique_once=True).to(DEV).train()
    points, feats, coors, fcl = points.to(DEV), feats.to(DEV), coors.to(DEV), fcl.to(DEV)
    _, group, out_coors = sir(points, feats, coors, fcl)
    head = MODELS.build(dict(CO.FSD_D1_HEAD, in_channel=group.shape[1], train_cfg=CO.FSD_D1_TRAIN_CFG)).to(DEV).train()
    cxyz = xyz_c.to(DEV)[out_coors[:, 2]]
    opt = torch.optim.Adam(list(sir.parameters()) + list(head.parameters()), lr=1e-3)
    Bd, Ld = [b.to(DEV) for b in Bx], [lab.to(DEV) for lab in L]
    totals = []
    for step in range(6):
        opt.zero_grad()
        _, group, oc = sir(points, feats, coors, fcl)
        out = head(group)
        losses = head.loss(out['cls_logits'], out['reg_preds'], cxyz, oc, Bd, Ld)
        loss = sum(losses.values())
        loss.backward()
        totals.append(loss.item())
        for n_, p in list(sir.named_parameters()) + list(head.named_parameters()):
            assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max().item() > 0, (step, n_)
        opt.step()
    print(f"[cluster_head] D1 SIR + head losses {['%.4f' % v for v in totals]}")
    assert totals[-1] < totals[0]
