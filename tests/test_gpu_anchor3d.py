"""GPU: Anchor3DHead's native training path (ops.anchor3d_targets, ops.anchor_focal_loss, ops.anchor_reg_dir_loss) against the reference's
own targets (tests/golden/anchor3d_targets.npz) and the CPU / float64 oracle (oracle/anchor3d_oracle.py), and the SECONDFPN +
Anchor3DHead modules built from the flagship config.

Targets: labels, weights, direction targets and num_total_pos bit-exact; every bbox_targets column bit-exact except the three log
columns, which lie within 2 ulp of the float64 log of the same fp32 ratio.  Covered: B = 1, 2, 5 with empty samples and an all-empty
batch; G = 1, 255, 256, 257 (around the kernel's 256-GT shared-memory chunk) and 4096, 4097 refused; duplicate GTs; anchors tied with one
GT under both gt_max_assign_all values; thresholds at an observed fp32 IoU and one ulp either side; min_pos_iou = 0; the nearest_bev
swap boundary, +-pi/2 and several periods out, the direction-bin boundaries +- 1 ulp (oracle/anchor3d_oracle.edge_yaws); GTs outside
the range and zero-width GTs; non-square and 1-cell-wide maps; assign_per_class; outputs pre-filled with NaN / 0xFF through the C ABI.

Losses: forward and backward against float64 autograd, with logits out to +-40, NaN logits and predictions, no positives, determinism
and no host sync.  Bounds (relative to the float64 value; gradients elementwise relative to the largest gradient) were set from the worst
error seen on an H100, with margin."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import anchor3d_oracle as AO
from oracle import iou3d_oracle as IO

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "anchor3d_targets.npz")
LOSS_TOL = 2e-7       # focal / L1 / direction loss, relative; worst seen 4.9e-8
GRAD_TOL = 1e-6       # gradients, max |err| / max |grad|; worst seen 3.6e-7


def _gen(geom):
    from sst_b200.anchor3d_modules import AlignedAnchor3DRangeGenerator
    g = dict(geom["head"]["anchor_generator"])
    g.pop("type")
    return AlignedAnchor3DRangeGenerator(**g)


def _native(geom, boxes, labels, **over):
    from sst_b200 import ops
    xc, yc, z, whl, rot = _gen(geom).axes((geom["H"], geom["W"]), DEV)
    asg = AO.assigner_args(geom)
    kw = dict(pos_iou_thr=[a["pos_iou_thr"] for a in asg], neg_iou_thr=[a["neg_iou_thr"] for a in asg],
              min_pos_iou=[a["min_pos_iou"] for a in asg], gt_max_assign_all=[a["gt_max_assign_all"] for a in asg],
              assign_per_class=geom["head"]["assign_per_class"], dir_offset=geom["head"]["dir_offset"])
    kw.update(over)
    return ops.anchor3d_targets(xc, yc, z, whl, rot, torch.cat(boxes).to(DEV), torch.cat(labels).to(DEV), [b.shape[0] for b in boxes],
                                geom["head"]["num_classes"], **kw)


def _oracle(geom, boxes, labels, assigners=None, assigned=None):
    anchors = AO.anchors_from_axes(*[t.cpu() for t in _gen(geom).axes((geom["H"], geom["W"]), DEV)])   # anchors copied from the device
    return AO.targets(anchors, boxes, labels, assigners or AO.assigner_args(geom), geom["head"]["num_classes"],
                      geom["head"]["assign_per_class"], geom["head"]["dir_offset"], assigned=assigned), anchors


def _log_ok(got, ref_anchor, gt, col):
    """|got - log(fp32 ratio)| <= 2 ulp of the float64 log"""
    ratio = (gt[:, col] / ref_anchor[:, col]).double()
    ref = torch.log(ratio)
    ulp = torch.from_numpy(np.spacing(ref.float().abs().numpy()).astype(np.float64))
    return bool(((got.double() == ref) | ((got.double() - ref).abs() <= 2 * ulp)).all())   # equal covers log(0) = -inf (zero-width GTs)


def _check(got, ref, anchors=None, boxes=None, assigned=None):
    names = ("labels", "label_weights", "bbox_targets", "bbox_weights", "dir_targets", "dir_weights")
    for k, name in enumerate(names):
        g = got[k].cpu()
        if name == "bbox_targets":
            assert torch.equal(g[..., [0, 1, 2, 6]], ref[k][..., [0, 1, 2, 6]]), "bbox_targets (x, y, z, yaw) differ"
            if anchors is None:
                ulp = (g[..., 3:6].view(torch.int32) - ref[k][..., 3:6].view(torch.int32)).abs().max().item()
                assert ulp <= 2, f"log columns off by {ulp} ulp"
            else:
                A = anchors.reshape(-1, 7)
                for b, gi in enumerate(assigned):
                    pos = torch.nonzero(gi >= 0)[:, 0]
                    if pos.numel():
                        for col in (3, 4, 5):
                            assert _log_ok(g[b, pos, col], A[pos], boxes[b][gi[pos]], col), f"log column {col} beyond 2 ulp"
                    neg = torch.nonzero(gi < 0)[:, 0]
                    assert not g[b, neg].any()
        else:
            assert torch.equal(g, ref[k]), f"{name} differs"
    assert int(got[6].item()) == int(ref[6]), f"num_total_pos {int(got[6].item())} != {int(ref[6])}"


@pytest.mark.parametrize("case", ["default", "per_class", "argmax_only"])
def test_targets_match_reference_golden(case):
    z = np.load(GOLDEN)
    kw = {"default": {}, "per_class": dict(assign_per_class=True), "argmax_only": dict(gt_max_assign_all=False)}[case]
    geom = AO.geometry(**kw)
    sizes = z[f"{case}/sizes"].tolist()
    boxes = list(torch.from_numpy(z[f"{case}/boxes"]).split(sizes))
    labels = list(torch.from_numpy(z[f"{case}/labels"]).split(sizes))
    got = _native(geom, boxes, labels)
    ref = tuple(torch.from_numpy(z[f"{case}/{k}"]) for k in ("labels_t", "label_weights", "bbox_targets", "bbox_weights", "dir_targets",
                                                             "dir_weights")) + (int(z[f"{case}/num_total_pos"]),)
    _check(got, ref)
    assert int((got[0] < geom["head"]["num_classes"]).sum()) > 20


CASES = [
    ("b1", {}, [40]), ("b2_empty", {}, [30, 0]), ("b5", {}, [12, 0, 1, 50, 7]), ("all_empty", {}, [0, 0]),
    ("g1", {}, [1]), ("g255", {}, [255, 3]), ("g256", {}, [256]), ("g257", {}, [2, 257]), ("g4096", {}, [4096]),
    ("argmax_only", dict(gt_max_assign_all=False), [80, 5]), ("per_class", dict(assign_per_class=True), [60, 0, 9]),
    ("per_class_argmax", dict(assign_per_class=True, gt_max_assign_all=False), [45]),
    ("min_pos_0", dict(thresholds=[(0.5, 0.3, 0.0)] * 3), [20, 4]),
    ("wide", dict(height=20, width=90), [50]), ("tall", dict(height=90, width=20), [50]),
    ("one_col", dict(height=60, width=1), [10]), ("one_row", dict(height=1, width=60), [10]),
    ("two_classes", dict(classes=(1, 2)), [30, 30]), ("one_size", dict(classes=(0,)), [25]),
]


@pytest.mark.parametrize("name,kw,sizes", CASES, ids=[c[0] for c in CASES])
def test_targets_match_oracle(name, kw, sizes):
    geom = AO.geometry(**kw)
    boxes, labels = AO.synth_batch(sum(map(ord, name)), geom, sizes)
    assigned = []
    ref, anchors = _oracle(geom, boxes, labels, assigned=assigned)
    got = _native(geom, boxes, labels)
    _check(got, ref, anchors, boxes, assigned)
    again = _native(geom, boxes, labels)
    for a, b in zip(got, again):
        assert torch.equal(a, b), "two calls differ"


def test_duplicates_and_ties():
    """an axis-aligned GT centred on a cell: the anchors of a size and rotation tie in IoU with it; a duplicate of it comes later.  The
    first copy wins the argmax rule, the last one the low-quality pass, under both gt_max_assign_all values"""
    for all_ in (True, False):
        geom = AO.geometry(gt_max_assign_all=all_)
        xc, yc, *_ = AO.axes(geom)
        g = torch.tensor([[float(xc[30]), float(yc[20]), 0.0, 2.08, 4.73, 1.77, 0.0]])
        g2 = torch.tensor([[float(xc[10]) + 0.32, float(yc[5]), 0.0, 0.84, 0.91, 1.74, 0.0]])   # on a cell edge: two cells tie
        boxes = [torch.cat([g, g2, g, g2])]
        labels = [torch.tensor([0, 2, 0, 2])]
        assigned = []
        ref, anchors = _oracle(geom, boxes, labels, assigned=assigned)
        got = _native(geom, boxes, labels)
        _check(got, ref, anchors, boxes, assigned)


def test_thresholds_at_observed_iou():
    geom = AO.geometry()
    boxes, labels = AO.synth_batch(5, geom, [40])
    ious = []
    anchors = AO.anchors_from_axes(*AO.axes(geom))
    AO.targets(anchors, boxes, labels, AO.assigner_args(geom), 3, ious=ious)
    v = ious[0][ious[0] > 0.2]
    picks = [float(v.min()), float(v.median()), float(v.max())]
    for iou in picks:
        for k in (-1, 0, 1):
            t = AO._ulp(iou, k)
            asg = [dict(pos_iou_thr=t, neg_iou_thr=t, min_pos_iou=t, gt_max_assign_all=True)] * 3
            assigned = []
            ref, anchors = _oracle(geom, boxes, labels, asg, assigned)
            got = _native(geom, boxes, labels, pos_iou_thr=[t] * 3, neg_iou_thr=[t] * 3, min_pos_iou=[t] * 3)
            _check(got, ref, anchors, boxes, assigned)


def test_refused_and_bad_arguments():
    from sst_b200 import _lib as L
    geom = AO.geometry(height=4, width=4)
    with pytest.raises(L.SSTB200Error, match="at most 4096"):
        _native(geom, *AO.synth_batch(1, geom, [4097]))
    with pytest.raises(L.SSTB200Error, match="at most 256"):
        _native(geom, *AO.synth_batch(1, geom, [0] * 257))
    with pytest.raises(L.SSTB200Error):
        _native(geom, [torch.zeros(3, 9)], [torch.zeros(3, dtype=torch.long)])


@pytest.mark.parametrize("fill", ["nan", "ff"])
def test_dirty_outputs_through_c_abi(fill):
    from sst_b200 import _lib as L
    geom = AO.geometry(height=30, width=25)
    boxes, labels = AO.synth_batch(3, geom, [30, 0, 8])
    ref = _native(geom, boxes, labels)
    outs = [torch.empty_like(t) for t in ref]
    for t in outs:
        if fill == "nan" and t.dtype == torch.float32:
            t.fill_(float("nan"))
        else:
            t.reshape(-1).view(torch.uint8).fill_(0xFF)
    xc, yc, z, whl, rot = _gen(geom).axes((geom["H"], geom["W"]), DEV)
    asg = AO.assigner_args(geom)
    gt, gl = torch.cat(boxes).to(DEV), torch.cat(labels).to(DEV)
    f = lambda k, ct: L.arr(ct, [a[k] for a in asg])  # noqa: E731
    c = L.ctx(DEV)
    L.check(c, L.lib().sstb200_anchor3d_targets(c, L.ptr(xc), xc.numel(), L.ptr(yc), yc.numel(), L.ptr(z), L.ptr(whl), 3, L.ptr(rot), 2,
                                                L.ptr(gt), L.ptr(gl), L.arr(C.c_int32, [0, 30, 30, 38]), 3, f("pos_iou_thr", C.c_float),
                                                f("neg_iou_thr", C.c_float), f("min_pos_iou", C.c_float), f("gt_max_assign_all", C.c_int32),
                                                0, 3, 0.7854, *[L.ptr(t) for t in outs]))
    for a, b in zip(outs, ref):
        assert torch.equal(a, b)


# ---- losses ----
def _loss_case(seed, sizes=(40, 0, 25), scale=1.0, geom=None):
    geom = geom or AO.geometry()
    boxes, labels = AO.synth_batch(seed, geom, list(sizes))
    tg = _native(geom, boxes, labels)
    cls, reg, dr = AO.synth_preds(seed, geom, len(sizes), scale)
    return geom, tg, cls, reg, dr


def _ref_losses(geom, tg, cls, reg, dr):
    t = [x.cpu() for x in tg]
    c64, r64, d64 = (x.double().requires_grad_(True) for x in (cls, reg, dr))
    C_ = geom["head"]["num_classes"]
    lc = AO.focal_loss(c64, t[0], t[1], int(t[6]), C_, 1.0)
    lb, ld = AO.reg_dir_loss(r64, d64, t[0], t[2], t[3], t[4], t[5], int(t[6]), C_, [1.0] * 7, 0.5, 0.2)
    return (lc, lb, ld), (c64, r64, d64)


def _native_losses(geom, tg, cls, reg, dr):
    from sst_b200 import ops
    cg, rg, dg = (x.to(DEV).requires_grad_(True) for x in (cls, reg, dr))
    C_ = geom["head"]["num_classes"]
    lc = ops.anchor_focal_loss(cg, tg[0], tg[1], tg[6], C_, 1.0)
    lb, ld = ops.anchor_reg_dir_loss(rg, dg, tg[0], tg[2], tg[3], tg[4], tg[5], tg[6], C_, [1.0] * 7, 0.5, 0.2)
    return (lc, lb, ld), (cg, rg, dg)


def _grad_err(got, ref):
    return ((got.cpu().double() - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("scale", [1.0, 20.0])
def test_losses_forward_backward(scale):
    """scale 20 puts logits out to about +-40 (the stable softplus form)"""
    geom, tg, cls, reg, dr = _loss_case(11, scale=scale)
    refs, r_in = _ref_losses(geom, tg, cls, reg, dr)
    gots, g_in = _native_losses(geom, tg, cls, reg, dr)
    for k, (g, r) in enumerate(zip(gots, refs)):
        err = abs(g.item() - r.item()) / abs(r.item())
        print(f"loss {k}: rel err {err:.2e}")
        assert err < LOSS_TOL, f"loss {k}: rel err {err}"
    sum(refs).backward()
    sum(gots).backward()
    for k, (g, r) in enumerate(zip(g_in, r_in)):
        err = _grad_err(g.grad, r.grad)
        print(f"grad {k}: err {err:.2e}")
        assert err < GRAD_TOL, f"grad {k}: err {err}"
    assert float(cls.abs().max()) > 30 or scale == 1.0


def test_no_positives_and_nan():
    from sst_b200 import ops
    geom, tg, cls, reg, dr = _loss_case(3, sizes=(0, 0))
    (lc, lb, ld), (cg, rg, dg) = _native_losses(geom, tg, cls, reg, dr)
    assert lb.item() == 0.0 and ld.item() == 0.0 and int(tg[6].item()) == 2
    (lc + lb + ld).backward()
    assert not rg.grad.any() and not dg.grad.any() and torch.isfinite(cg.grad).all()
    # NaN logit: loss NaN, gradient NaN at that element only; NaN box prediction at a positive: loss_bbox NaN
    geom, tg, cls, reg, dr = _loss_case(4, sizes=(30,))
    cls[0, 5, 3, 4] = float("nan")
    pos = torch.nonzero(tg[0][0].cpu() < 3)[0, 0].item()
    hw, a = divmod(pos, 6)
    reg[0, a * 7 + 2, hw // 60, hw % 60] = float("nan")
    (lc, lb, ld), (cg, rg, dg) = _native_losses(geom, tg, cls, reg, dr)
    assert torch.isnan(lc) and torch.isnan(lb) and torch.isfinite(ld)
    lc.backward()
    nan = torch.isnan(cg.grad)
    assert nan.sum().item() == 1 and nan[0, 5, 3, 4]
    assert ops is not None


def test_losses_deterministic_and_no_host_sync():
    geom, tg, cls, reg, dr = _loss_case(8)
    runs = []
    for _ in range(2):
        (lc, lb, ld), ins = _native_losses(geom, tg, cls, reg, dr)
        (lc + lb + ld).backward()
        runs.append([lc, lb, ld] + [x.grad for x in ins])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    from sst_b200 import ops
    cg = cls.to(DEV).requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = ops.anchor_focal_loss(cg, tg[0], tg[1], tg[6], 3, 1.0)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


# ---- modules ----
def _flagship_head(H=64, W=48):
    from sst_b200 import flagship as fl
    from sst_b200.registry import MODELS
    neck = MODELS.build(fl.ANCHOR_NECK).to(DEV)
    head = MODELS.build(dict(fl.ANCHOR_HEAD, train_cfg=fl.ANCHOR_TRAIN_CFG, test_cfg=fl.ANCHOR_TEST_CFG)).to(DEV)
    neck.init_weights()
    head.init_weights()
    return neck, head


def test_flagship_neck_and_head_train_step():
    torch.manual_seed(0)
    neck, head = _flagship_head()
    x = torch.randn(2, 128, 64, 48, device=DEV, requires_grad=True)
    feats = neck([x])
    cls, reg, dr = head(feats)
    assert cls[0].shape == (2, 18, 64, 48) and reg[0].shape == (2, 42, 64, 48) and dr[0].shape == (2, 12, 64, 48)
    # boxes inside the first 64 x 48 cells of the 468 x 468 range
    g = torch.Generator().manual_seed(1)
    n = 30
    ctr = torch.stack([-74.88 + torch.rand(n, generator=g) * 48 * 0.32, -74.88 + torch.rand(n, generator=g) * 64 * 0.32], 1)
    lab = torch.randint(0, 3, (n,), generator=g)
    size = torch.tensor([[2.08, 4.73, 1.77], [0.84, 1.81, 1.77], [0.84, 0.91, 1.74]])[lab]
    boxes = torch.cat([ctr, torch.zeros(n, 1), size, torch.rand(n, 1, generator=g) * 6 - 3], 1)
    losses = head.loss(cls, reg, dr, [boxes, boxes[:10].to(DEV)], [lab, lab[:10]], None)
    total = sum(v[0] for v in losses.values())
    total.backward()
    assert all(torch.isfinite(v[0]) for v in losses.values()) and losses["loss_bbox"][0].item() > 0
    assert torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0


@pytest.mark.parametrize("classes", [(1, 2), (0, 1, 2)])
def test_get_bboxes_matches_oracle(classes):
    from sst_b200.registry import MODELS
    geom = AO.geometry(height=50, width=70, classes=classes)
    head = MODELS.build(dict(geom["head"], type="Anchor3DHead", train_cfg=geom["train_cfg"], test_cfg=dict(geom["test_cfg"], nms_pre=1500)))
    cls, reg, dr = AO.synth_preds(21, geom, 2)
    anchors = AO.anchors_from_axes(*AO.axes(geom)).reshape(-1, 7)
    got = head.get_bboxes([cls.to(DEV)], [reg.to(DEV)], [dr.to(DEV)], [{}, {}])
    for b in range(2):
        ref = AO.get_bboxes_single(cls[b], reg[b], dr[b], anchors, len(classes), dict(geom["test_cfg"], nms_pre=1500))
        assert ref[0].shape[0] > 0
        # the same detections; two boxes of one class whose scores differ by an ulp between the GPU's and the CPU's sigmoid may trade
        # places, so both lists are compared in (label, score) order
        rows = [torch.cat([r[2].cpu().double()[:, None], r[1].cpu().double()[:, None], r[0].cpu().double()], 1) for r in (got[b], ref)]
        assert rows[0].shape == rows[1].shape
        rows = [r[torch.from_numpy(np.lexsort((-r[:, 1].numpy(), r[:, 0].numpy())))] for r in rows]
        torch.testing.assert_close(rows[0], rows[1], rtol=1e-5, atol=1e-5)


def test_unsupported_settings_raise():
    from sst_b200.anchor3d_modules import Anchor3DHead
    geom = AO.geometry()
    base = dict(geom["head"], train_cfg=geom["train_cfg"], test_cfg=geom["test_cfg"])
    gen = geom["head"]["anchor_generator"]
    bad = [dict(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=True)), dict(loss_cls=dict(type='FocalLoss', use_sigmoid=False)),
           dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=3.0)), dict(loss_bbox=dict(type='SmoothL1Loss')),
           dict(loss_dir=dict(type='CrossEntropyLoss', use_sigmoid=True)), dict(use_direction_classifier=False),
           dict(diff_rad_by_sin=False), dict(bbox_coder=dict(type='DeltaXYZWLHRBBoxCoder', code_size=9)),
           dict(anchor_generator=dict(gen, type='Anchor3DRangeGenerator')), dict(anchor_generator=dict(gen, align_corner=True)),
           dict(anchor_generator=dict(gen, custom_values=[0, 0])),
           dict(train_cfg=dict(geom["train_cfg"], assigner=geom["train_cfg"]["assigner"][0])),
           dict(train_cfg=dict(geom["train_cfg"], assigner=geom["train_cfg"]["assigner"][:2])),
           dict(train_cfg=dict(geom["train_cfg"], assigner=[dict(a, ignore_iof_thr=0.5) for a in geom["train_cfg"]["assigner"]])),
           dict(train_cfg=dict(geom["train_cfg"], assigner=[dict(a, iou_calculator=dict(type='BboxOverlaps3D', coordinate='lidar'))
                                                            for a in geom["train_cfg"]["assigner"]])),
           dict(train_cfg=dict(geom["train_cfg"], pos_weight=2.0))]
    for over in bad:
        with pytest.raises(ValueError):
            Anchor3DHead(**dict(base, **over))
    head = Anchor3DHead(**dict(base, test_cfg=dict(geom["test_cfg"], wnms=True))).to(DEV)
    cls, reg, dr = AO.synth_preds(1, geom, 1)
    with pytest.raises(NotImplementedError):
        head.get_bboxes([cls.to(DEV)], [reg.to(DEV)], [dr.to(DEV)], [{}])
    assert IO is not None
