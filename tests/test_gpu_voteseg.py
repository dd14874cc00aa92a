"""GPU: VoteSegHead's native training path (ops.voteseg_targets, ops.voteseg_loss) against the reference's own targets
(tests/golden/voteseg_targets.npz) and the CPU / float64 oracle (oracle/voteseg_oracle.py), the VoteSegHead module, and a VoteSegmentor
built from the D1 config training on synthetic Waymo-shaped sweeps.

Targets: labels, vote targets and mask bit-exact.  Covered: B = 1, 2, 3, 8 with zero-point and zero-GT samples; G = 1, 255, 256, 257,
512 (around the kernel's 256-GT shared-memory chunk) and the 4096 cap, 4097 refused; an invalid-label box of lower index overlapping a
valid one; points on the box faces and one ulp either side; yaws of +-pi; outputs pre-filled with NaN / 0xFF through the C ABI.

Losses: forward and backward against float64 autograd, sigmoid focal (C = 1, 3) and softmax cross-entropy (C = 10 + 1, 26 + 1), with
logits out to +-40, logit_scale != 1 and class weights; NaN logits, NaN vote predictions and no valid point; two-run bit identity; no
host sync.  Metrics: counts exact against the oracle.  The fp32 scores on the GPU and the oracle's float64 scores differ by about 1e-7, so
the generated logits keep every score at least 1e-5 from its threshold (oracle.voteseg_oracle.clear_of_thresholds): a score closer than
that could compare differently in the two precisions, and the counts would then differ for a reason that is not an error.  Bounds
(relative to the float64 value; gradients elementwise relative to the largest gradient) were set from the worst error seen on an H100,
with margin."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from oracle import voteseg_oracle as VO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "voteseg_targets.npz")
LOSS_TOL = 3e-7       # loss_sem_seg / loss_vote, relative; worst seen 7.1e-8
GRAD_TOL = 2e-6       # gradients, max |err| / max |grad|; worst seen 4.5e-7


def _targets(P, B, L, num_classes):
    from sst_b200 import ops
    return ops.voteseg_targets([p.to(DEV) for p in P], None, [b.to(DEV) for b in B], [lab.to(DEV) for lab in L], num_classes)


def _equal(got, ref):
    for a, b in zip(got, ref):
        assert a.dtype == b.dtype and torch.equal(a.cpu(), b)


# ---- targets ----
def test_targets_match_golden_reference():
    from sst_b200 import ops
    g = np.load(GOLDEN)
    for name in ("waymo", "nusc"):
        pts = torch.from_numpy(g[f"{name}/points"]).to(DEV)
        offs = np.concatenate([[0], np.cumsum(g[f"{name}/point_sizes"])]).tolist()
        boxes, labels = torch.from_numpy(g[f"{name}/boxes"]), torch.from_numpy(g[f"{name}/labels"])
        bo = np.concatenate([[0], np.cumsum(g[f"{name}/box_sizes"])]).tolist()
        B = [boxes[a:b].to(DEV) for a, b in zip(bo, bo[1:])]
        L = [labels[a:b].to(DEV) for a, b in zip(bo, bo[1:])]
        got = ops.voteseg_targets(pts, offs, B, L, int(g[f"{name}/num_classes"]))
        ref = [torch.from_numpy(g[f"{name}/{k}"]) for k in ("labels_t", "vote_targets", "vote_mask")]
        assert torch.equal(got[0].cpu(), ref[0]) and torch.equal(got[2].cpu(), ref[2])
        # the golden vote targets come from the reference run on the CPU, whose vectorised square root can be one ulp off the correctly
        # rounded one the GPU (and torch's `** 0.5` there) gives: within one ulp of it, bit-exact against the oracle's IEEE square root
        ulp = (got[1].cpu().view(torch.int32).long() - ref[1].view(torch.int32).long()).abs().max().item()
        assert ulp <= 1, ulp
        P = [pts.cpu()[a:b] for a, b in zip(offs, offs[1:])]
        _equal(got, VO.targets(P, [b.cpu() for b in B], [lab.cpu() for lab in L], int(g[f"{name}/num_classes"])))


@pytest.mark.parametrize("sizes", [([900], [20]), ([0, 700], [5, 12]), ([1200, 300, 0], [30, 0, 7]),
                                   ([500, 0, 800, 300, 0, 1000, 20, 400], [10, 3, 0, 25, 0, 40, 2, 9])],
                         ids=["B1", "B2", "B3", "B8"])
def test_targets_match_oracle(sizes):
    n_points, n_boxes = sizes
    P, B, L = VO.synth_batch(len(n_points) * 31, n_points, n_boxes, 3)
    for b in range(len(P)):
        if n_points[b] and n_boxes[b] >= 3:
            P[b] = torch.cat([P[b], torch.nn.functional.pad(VO.face_points(B[b][:3]), (0, 2))])
            B[b][1], L[b][0], L[b][1] = B[b][0], -1, 2          # an invalid box of lower index on top of a valid one
    _equal(_targets(P, B, L, 3), VO.targets(P, B, L, 3))


@pytest.mark.parametrize("G", [1, 255, 256, 257, 512, 4096])
def test_targets_gt_chunk_edges(G):
    g = torch.Generator().manual_seed(G)
    boxes, lab = VO.synth_boxes(g, G, 3, spread=30.0)
    pts = VO.points_around(g, boxes, 3000, spread=30.0)
    # points inside the last boxes only: the scan has to reach the last chunk
    pts = torch.cat([pts, VO.points_around(g, boxes[-3:], 60, spread=30.0, inside=1.0)])
    P, B, L = [pts, pts[:100]], [boxes, boxes[:0]], [lab, lab[:0]]
    _equal(_targets(P, B, L, 3), VO.targets(P, B, L, 3))


def test_targets_refuse_more_than_the_gt_cap():
    from sst_b200 import _lib
    g = torch.Generator().manual_seed(1)
    boxes, lab = VO.synth_boxes(g, 4097, 3)
    with pytest.raises(_lib.SSTB200Error, match="at most 4096"):
        _targets([torch.zeros(10, 3)], [boxes], [lab], 3)


def test_targets_yaw_pi_and_dirty_outputs_through_c_abi():
    from sst_b200 import _lib as L
    g = torch.Generator().manual_seed(5)
    boxes, lab = VO.synth_boxes(g, 40, 3, spread=15.0)
    boxes[:20, 6] = torch.tensor([math.pi, -math.pi] * 10, dtype=torch.float32)
    pts = torch.cat([VO.points_around(g, boxes, 4000, spread=15.0, cols=4), torch.nn.functional.pad(VO.face_points(boxes[:20]), (0, 1))])
    ref = VO.targets([pts[:2500], pts[2500:]], [boxes[:25], boxes[25:]], [lab[:25], lab[25:]], 3)
    p, bx, lb = pts.to(DEV), boxes.to(DEV), lab.to(DEV)
    N = pts.shape[0]
    labels = torch.full((N,), -7, dtype=torch.int64, device=DEV)
    vt = torch.full((N, 3), float("nan"), device=DEV)
    mask = torch.full((N,), 0xFF, dtype=torch.uint8, device=DEV)
    c = L.ctx(DEV)
    L.check(c, L.lib().sstb200_voteseg_targets(c, p.data_ptr(), 4, L.arr(C.c_int32, [0, 2500, N]), bx.data_ptr(), lb.data_ptr(),
                                               L.arr(C.c_int32, [0, 25, 40]), 2, 3, labels.data_ptr(), vt.data_ptr(), mask.data_ptr()))
    _equal((labels, vt, mask.bool()), ref)
    assert set(mask.unique().tolist()) <= {0, 1}


# ---- losses ----
def _frame(mode, seed, n_points=(1500, 0, 900), n_boxes=(30, 4, 0), wide=False):
    m = VO.LOSS_MODES[mode]
    P, B, L = VO.synth_batch(seed, list(n_points), list(n_boxes), m["num_classes"])
    t = VO.targets(P, B, L, m["num_classes"])
    Cn = m["num_classes"] + (0 if m["loss_decode"]["type"] == "FocalLoss" else 1)
    x, v = VO.synth_preds(seed, t[0].shape[0], Cn, scale=4.0)
    if wide:
        x[::13] = 40.0 * torch.sign(torch.randn(x[::13].shape, generator=torch.Generator().manual_seed(seed)))
    x = VO.clear_of_thresholds(x, VO.loss_kwargs(mode), seed=seed)
    return t, x, v


def _native(mode, t, x, v, strided=False):
    from sst_b200 import ops
    kw = dict(VO.loss_kwargs(mode), num_classes=x.shape[1])
    if strided:          # rows read in place with a row stride: the two heads as column blocks of one tensor
        both = torch.cat([x, v], 1).to(DEV).requires_grad_(True)
        xg, vg = both[:, :x.shape[1]], both[:, x.shape[1]:]
        leaf = both
    else:
        xg, vg = x.to(DEV).requires_grad_(True), v.to(DEV).requires_grad_(True)
        leaf = None
    seg, vote, met = ops.voteseg_loss(xg, vg, *[a.to(DEV) for a in t], **kw)
    return seg, vote, met, xg, vg, leaf


def _oracle(mode, t, x, v):
    xo, vo = x.double().requires_grad_(True), v.double().requires_grad_(True)
    seg, vote = VO.losses(xo, vo, *t, **VO.loss_kwargs(mode))
    return seg, vote, xo, vo


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-30)


def _grel(g, ref):
    return (g.detach().cpu().double() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


@pytest.mark.parametrize("mode", list(VO.LOSS_MODES))
@pytest.mark.parametrize("wide", [False, True], ids=["randn", "pm40"])
def test_losses_and_gradients_match_float64(mode, wide):
    t, x, v = _frame(mode, 11 + sum(map(ord, mode)), wide=wide)
    seg, vote, met, xg, vg, _ = _native(mode, t, x, v)
    (0.6 * seg + 1.3 * vote).backward()
    rs, rv, xo, vo = _oracle(mode, t, x, v)
    (0.6 * rs + 1.3 * rv).backward()
    errs = [_rel(seg.item(), rs.item()), _rel(vote.item(), rv.item())]
    gerrs = [_grel(xg.grad, xo.grad), _grel(vg.grad, vo.grad)]
    print(f"[voteseg] {mode} wide={wide}: loss rel err {max(errs):.2e}, grad rel err {max(gerrs):.2e}")
    assert max(errs) < LOSS_TOL and max(gerrs) < GRAD_TOL, (errs, gerrs)
    ref = VO.metrics(x, t[0], **VO.loss_kwargs(mode))
    assert list(met) == list(ref)
    for k in ref:
        assert torch.equal(met[k].cpu(), ref[k]), k


def test_losses_read_strided_rows_in_place():
    t, x, v = _frame("nusc_ce", 4)
    seg, vote, _, xg, vg, leaf = _native("nusc_ce", t, x, v, strided=True)
    (seg + vote).backward()
    rs, rv, xo, vo = _oracle("nusc_ce", t, x, v)
    (rs + rv).backward()
    assert _rel(seg.item(), rs.item()) < LOSS_TOL and _rel(vote.item(), rv.item()) < LOSS_TOL
    assert _grel(leaf.grad, torch.cat([xo.grad, vo.grad], 1)) < GRAD_TOL


@pytest.mark.parametrize("mode", ["waymo_focal", "nusc_ce"])
def test_nan_logit_poisons_only_its_own_gradient(mode):
    t, x, v = _frame(mode, 21)
    r = 7
    xn = x.clone()
    xn[r, 0] = float("nan")
    seg, vote, _, xg, vg, _ = _native(mode, t, xn, v)
    (seg + vote).backward()
    assert math.isnan(seg.item()) and not math.isnan(vote.item())
    rs, rv, xo, vo = _oracle(mode, t, x, v)
    (rs + rv).backward()
    g = xg.grad.cpu().double()
    bad = torch.zeros_like(g, dtype=torch.bool)
    if mode == "waymo_focal":
        bad[r, 0] = True
    else:
        bad[r] = True                       # softmax: the whole row goes through logsumexp
    assert g[bad].isnan().all() and not g[~bad].isnan().any()
    assert (g[~bad] - xo.grad[~bad]).abs().max().item() < GRAD_TOL * xo.grad.abs().max().item()
    assert _grel(vg.grad, vo.grad) < GRAD_TOL


def test_nan_vote_prediction():
    t, x, v = _frame("waymo_focal", 22)
    i = int(torch.nonzero(t[2])[0])
    ch = 3 * int(t[0][i])
    j = int(torch.nonzero(t[2])[1])
    vn = v.clone()
    vn[i, ch] = float("nan")                               # read by the loss
    vn[j, (3 * int(t[0][j]) + 3) % 9] = float("nan")       # another class's channel of a valid point: never read
    seg, vote, _, xg, vg, _ = _native("waymo_focal", t, x, vn)
    (seg + vote).backward()
    rs, rv, xo, vo = _oracle("waymo_focal", t, x, vn)
    (rs + rv).backward()
    assert math.isnan(vote.item()) and math.isnan(rv.item()) and not math.isnan(seg.item())
    assert torch.equal(vg.grad.cpu().double().isnan(), vo.grad.isnan()) and not vg.grad.isnan().any()
    assert _grel(vg.grad, vo.grad) < GRAD_TOL
    # NaN only in channels the loss never reads (other classes, background points): the loss stays finite and equal to float64
    vn = v.clone()
    vn[j, (3 * int(t[0][j]) + 3) % 9] = float("nan")
    vn[int(torch.nonzero(~t[2])[0])] = float("nan")
    _, vote, _, _, _, _ = _native("waymo_focal", t, x, vn)
    _, rv, _, _ = _oracle("waymo_focal", t, x, vn)
    assert not math.isnan(vote.item()) and _rel(vote.item(), rv.item()) < LOSS_TOL


def test_no_valid_point():
    t, x, v = _frame("waymo_focal", 23)
    labels, mask = torch.full_like(t[0], 3), torch.zeros_like(t[2])
    for bad in (None, float("inf"), float("nan")):
        vv = v.clone()
        if bad is not None:
            vv[3, 5] = bad
        seg, vote, met, xg, vg, _ = _native("waymo_focal", (labels, t[1], mask), x, vv)
        (seg + vote).backward()
        assert (bad is None and vote.item() == 0.0) or (bad is not None and math.isnan(vote.item()))
        assert torch.count_nonzero(vg.grad).item() == 0
        rs, _, xo, _ = _oracle("waymo_focal", (labels, t[1], mask), x, vv)
        rs.backward()
        assert _rel(seg.item(), rs.item()) < LOSS_TOL and _grel(xg.grad, xo.grad) < GRAD_TOL
        assert all(met[k].item() == 0.0 for k in met)


def test_two_runs_are_bit_identical():
    t, x, v = _frame("argo_ce", 31, n_points=(20000, 15000), n_boxes=(80, 60))
    outs = []
    for _ in range(2):
        seg, vote, met, xg, vg, _ = _native("argo_ce", t, x, v)
        (seg + vote).backward()
        outs.append([seg.detach(), vote.detach(), xg.grad, vg.grad] + [met[k] for k in met])
    for a, b in zip(*outs):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


def test_no_host_sync():
    from sst_b200 import ops
    P, B, L = VO.synth_batch(3, [3000, 2000], [30, 20], 3)
    pts, bx, lb = [p.to(DEV) for p in P], [b.to(DEV) for b in B], [lab.to(DEV) for lab in L]
    x, v = (a.to(DEV).requires_grad_(True) for a in VO.synth_preds(3, 5000, 3))
    cfg = ops.VoteSegLossConfig(3, True, **{k: w for k, w in VO.loss_kwargs("waymo_focal").items() if k != "use_sigmoid"})
    # warm-up: the loss forward carves its block partials from the context arena, and growing the arena is a cudaMalloc, which
    # set_sync_debug_mode does not see; the checked calls below are the steady state of a training loop
    seg, vote, _ = ops.voteseg_loss(x, v, *ops.voteseg_targets(pts, None, bx, lb, 3), cfg)
    (seg + vote).backward()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t = ops.voteseg_targets(pts, None, bx, lb, 3)
        seg, vote, met = ops.voteseg_loss(x, v, *t, cfg)
        (seg + vote).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert set(met) == {"recall_Car", "recall_Ped", "recall_Cyc"}


# ---- modules ----
@pytest.mark.parametrize("mode", ["waymo_focal", "argo_ce"])
def test_head_forward_train_matches_oracle_head(mode):
    """VoteSegHead.forward_train on the GPU against the same head in float64 on the CPU (torch MLP, plain BN) with the oracle's losses
    (pinned to the reference's own `losses` by tests/test_oracle_voteseg_vs_reference.py): losses, training-log metrics, parameter and
    input gradients"""
    from sst_b200.registry import MODELS
    cfg, train_cfg = VO.head_cfg(mode), VO.LOSS_MODES[mode]["train_cfg"]
    torch.manual_seed(2)
    mine = MODELS.build(cfg)
    ref = MODELS.build(dict(cfg, norm_cfg=dict(type="BN1d")))          # single process: naiveSyncBN1d is BN1d
    ref.load_state_dict(mine.state_dict())
    ref = ref.double().train()
    mine.train_cfg = train_cfg
    mine = mine.to(DEV).train()
    t, _, _ = _frame(mode, 41)
    feats = torch.randn((t[0].shape[0], 16), generator=torch.Generator().manual_seed(41))
    fo, fg = feats.double().requires_grad_(True), feats.to(DEV).requires_grad_(True)
    x, v = ref.forward(fo)
    rs, rv = VO.losses(x, v, *t, **VO.loss_kwargs(mode))
    lm = mine.forward_train(fg, None, *[a.to(DEV) for a in t])
    (rs + rv).backward()
    (lm["loss_sem_seg"] + lm["loss_vote"]).backward()
    assert _rel(lm["loss_sem_seg"].item(), rs.item()) < 1e-4 and _rel(lm["loss_vote"].item(), rv.item()) < 1e-4
    assert _grel(fg.grad, fo.grad) < 1e-4
    rp = dict(ref.named_parameters())
    for n, p in mine.named_parameters():
        assert _grel(p.grad, rp[n].grad) < 1e-4, n
    # the metrics of the logits this head produced; every score is far enough from its threshold that fp32 and float64 agree
    met = {k: w for k, w in lm.items() if k.startswith("recall_") or k == "num_fg"}
    logits = mine.forward(fg.detach())[0].detach().cpu()
    thr = torch.tensor(train_cfg["score_thresh"], dtype=torch.float64)
    assert (VO.scores(logits, **VO.loss_kwargs(mode)) - thr).abs().min().item() > 1e-6
    ref_met = VO.metrics(logits, t[0], **VO.loss_kwargs(mode))
    assert list(met) == list(ref_met)
    for k in ref_met:
        assert torch.equal(met[k].cpu(), ref_met[k]), k


def test_refused_settings_raise():
    from sst_b200.voteseg_modules import VoteSegHead
    base = VO.head_cfg("waymo_focal")
    base.pop("type")
    for kw in (dict(loss_aux=dict(type="LovaszLoss")), dict(loss_decode=dict(type="FocalLoss", use_sigmoid=True, gamma=0.5)),
               dict(loss_decode=dict(type="FocalLoss", gamma=2.0, alpha=0.25)),       # use_sigmoid missing: read as False by the head
               dict(loss_decode=dict(type="DiceLoss")), dict(loss_vote=dict(type="SmoothL1Loss"))):
        with pytest.raises(ValueError):
            VoteSegHead(**dict(base, **kw))
    head = VoteSegHead(**base)
    for cfg in (dict(centroid_offset=True), dict(extra_width=0.1)):
        with pytest.raises(ValueError):
            head.train_cfg = cfg


# ---- training ----
def test_d1_segmentor_trains():
    """A few Adam steps of the D1 VoteSegmentor on synthetic Waymo-shaped sweeps: the loss decreases, every head and front parameter
    gets a non-zero gradient at every step; at the first step the head's parameter and input gradients agree with the oracle head
    (float64, the same weights) run on the same features."""
    from sst_b200.registry import MODELS
    torch.manual_seed(0)
    cfg = dict(VO.FSD_D1_SEGMENTOR)
    seg = MODELS.build(cfg).to(DEV).train()
    seg.segmentation_head.init_weights()
    P, B, L = VO.waymo_sweeps(3, 2, 30000, 40)
    pts, bx, lb = [p.to(DEV) for p in P], [b.to(DEV) for b in B], [lab.to(DEV) for lab in L]
    opt = torch.optim.Adam(seg.parameters(), lr=2e-3)
    totals = []
    for step in range(5):
        opt.zero_grad()
        out = seg.forward_train(pts, None, bx, lb, as_subsegmentor=True)
        feats = out["seg_feats"]
        feats.retain_grad()
        loss = out["losses"]["loss_sem_seg"] + out["losses"]["loss_vote"]
        loss.backward()
        totals.append(loss.item())
        for name, p in seg.named_parameters():
            assert p.grad is not None and p.grad.abs().max().item() > 0, (step, name)
        if step == 0:
            _check_head_against_oracle(seg.segmentation_head, out, P, B, L, feats)
        opt.step()
    print(f"[voteseg] D1 segmentor losses {['%.4f' % v for v in totals]}")
    assert totals[-1] < totals[0]
    assert set(out["losses"]) == {"loss_sem_seg", "loss_vote", "recall_Car", "recall_Ped", "recall_Cyc"}


def _check_head_against_oracle(head, out, P, B, L, feats):
    """the head's parameter and input gradients against float64 autograd through an oracle head (torch MLP + oracle losses)"""
    from sst_b200.voteseg_modules import VoteSegHead
    pts, bidx = out["seg_points"].cpu(), out["batch_idx"].cpu()
    # the points the neck keeps, in order: a point's targets depend on the point alone
    t = VO.targets([pts[bidx == b] for b in range(len(P))], B, L, 3)
    hc = dict(VO.FSD_D1_SEGMENTOR["segmentation_head"], norm_cfg=dict(type="BN1d"))   # single process: naiveSyncBN1d is BN1d
    hc.pop("type")
    ref = VoteSegHead(**hc)
    ref.load_state_dict(head.state_dict())
    ref = ref.double().train()
    fo = feats.detach().cpu().double().requires_grad_(True)
    x, v = ref.forward(fo)
    rs, rv = VO.losses(x, v, *t, **dict(VO.WAYMO_CFG, loss_weight=1.0, loss_weight_vote=1.0))
    (rs + rv).backward()
    assert _rel(out["losses"]["loss_sem_seg"].item(), rs.item()) < 1e-4
    assert _rel(out["losses"]["loss_vote"].item(), rv.item()) < 1e-4
    assert _grel(feats.grad, fo.grad) < 1e-3
    rp = dict(ref.named_parameters())
    for n, p in head.named_parameters():
        assert _grel(p.grad, rp[n].grad) < 1e-3, n
