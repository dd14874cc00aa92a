"""CPU: oracle/roi_head_oracle.py against the reference's own FSD second stage (fsd_roi_head.py's _assign_and_sample, the whole
FullySparseBboxHead of fsd_bbox_head.py and IoUNegPiecewiseSampler, compiled unmodified through oracle/roi_head_ref.py with mmdet 2.14's
MaxIoUAssigner, RandomSampler and SamplingResult restated and random_choice following the key rule): sampled indices, GT rows and
labels equal; box targets within 1e-12 in float64 and within the reference's own fp32 rounding in float32; losses within 1e-12 in float64; get_bboxes equal; the golden file's
contents; and for every config that declares the stage, state-dict keys and shapes equal to the reference head's."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_roi_head as MG
from oracle import roi_head_oracle as RO
from oracle import roi_head_ref as RR

pytestmark = pytest.mark.skipif(not RR.available(), reason="reference tree not present")

CONFIGS = ["fsd/fsd_waymoD1_1x.py", "fsd/fsd_waymoD1_1x_3f.py", "fsd/fsd_waymoD1_1x_sst_encoder.py", "fsd/fsd_waymoD1_1x_submission.py",
           "fsdv2/fsdv2_waymo_1x.py", "fsdv2/fsdv2_waymo_2x.py"]
ASSIGNERS = MG.ASSIGNERS


@pytest.mark.parametrize("per_class", [True, False])
def test_assign_and_sample_match_reference(per_class):
    N = RR.load_roi_head()
    cfg = MG.train_cfg(per_class=per_class, num=128)
    batch = MG.batch([(300, 60), (0, 20), (200, 50), (80, 0)], seed=4)
    keys = [torch.rand(max(len(p), 1), generator=torch.Generator().manual_seed(10 + b), dtype=torch.float64)
            for b, (p, _, _, _) in enumerate(batch)]
    props = [(N.Boxes(p.double()), torch.rand(len(p)), l) for p, l, _, _ in batch]
    res = N.assign_and_sample(cfg, props, [N.Boxes(g.double()) for _, _, g, _ in batch], [l for _, _, _, l in batch], keys)
    for b, ((p, l, g, gl), r) in enumerate(zip(batch, res)):
        if len(p) == 0:   # the reference's fake box
            p, l = torch.tensor([[0, 0, 5, 1, 1, 1, 0]], dtype=torch.float32), torch.tensor([0])
        inds, iou, rows, lab, npos = RO.assign_and_sample(p, l, keys[b], g, gl, ASSIGNERS if per_class else ASSIGNERS[:1], per_class,
                                                          128, 0.55, [0.8, 0.2], [0.55, 0.1])
        assert torch.equal(inds, torch.cat([r.pos_inds, r.neg_inds])), b
        assert npos == len(r.pos_inds)
        assert torch.equal(rows[:npos], r.pos_assigned_gt_inds)
        assert torch.equal(lab[:npos], r.pos_gt_labels)
        assert torch.equal(iou, r.iou)


def test_targets_and_losses_match_reference():
    N = RR.load_roi_head()
    cfg = RR.Cfg(MG.train_cfg())
    head = N.build_head(MG.small_head(), cfg)
    inp = MG.golden_inputs(seed=7)
    res = MG.reference_sampling(N, cfg, inp, dtype=torch.float64)
    for r in res:   # get_multi_class_soft_label writes fp32 labels: it takes the IoU in fp32, as in training
        r.iou = r.iou.float()
    t = head.get_targets(res, cfg)
    label, bbox_targets, bidx, pos_gt, pos_lab, reg_mask, lw, bw = t
    soft, bt_rows, pg_rows, lab_rows = [], [], [], []
    for r in res:
        s, bt = RO.targets(r.bboxes, r.iou.double(), r.pos_gt_bboxes, r.pos_gt_labels, MG.POS_THR, MG.NEG_THR)
        soft.append(s), bt_rows.append(bt)
    assert (torch.cat(soft) - label.double()).abs().max().item() < 1e-6
    assert (torch.cat(bt_rows) - bbox_targets).abs().max().item() < 1e-12
    # float32: the reference's own fp32 chain against the oracle's float64 rounded once
    res32 = MG.reference_sampling(N, cfg, inp, dtype=torch.float32)
    t32 = head.get_targets(res32, cfg)
    bt64 = torch.cat([RO.targets(r.bboxes.double(), r.iou.double(), r.pos_gt_bboxes.double(), r.pos_gt_labels, MG.POS_THR,
                                   MG.NEG_THR)[1] for r in res32])
    # translate / rotate / encode are a few fp32 roundings in the reference, with cancellation near 0: an absolute bound of a few fp32 eps
    assert ((t32[1].double() - bt64).abs() <= 2e-6 * (1 + bt64.abs())).all()
    # losses, float64, with empty RoIs
    R = len(label)
    g = torch.Generator().manual_seed(3)
    rois = torch.cat([torch.cat([torch.full((len(r.bboxes), 1), float(b), dtype=torch.float64), r.bboxes], 1) for b, r in enumerate(res)])
    cls = (torch.randn(R, 1, generator=g, dtype=torch.float64) * 2).requires_grad_()
    pred = (torch.randn(R, 7, generator=g, dtype=torch.float64) * 0.3).requires_grad_()
    nonempty = torch.rand(R, generator=g) > 0.15
    head.train_cfg = RR.Cfg(dict(cfg, sync_cls_avg_factor=False, sync_reg_avg_factor=False))   # keep the factors float64
    ref = head.loss(cls, pred, nonempty, rois, label.clone(), bbox_targets, bidx, pos_gt, pos_lab, reg_mask.clone(), lw.clone(), bw.clone())
    rows = torch.nonzero(reg_mask > 0).view(-1)
    dense = lambda v, w: torch.zeros((R,) + v.shape[1:], dtype=v.dtype).index_copy(0, rows, v) if w is None else \
        torch.full((R,), w, dtype=v.dtype).index_copy(0, rows, v)  # noqa: E731
    mine = RO.losses(cls, pred, nonempty, label, reg_mask, dense(bbox_targets, None), dense(pos_gt[:, :7], None), dense(pos_lab, -1),
                     rois[:, 1:], dict(w_cls=1.0, w_bbox=2.0, smooth_l1=False, beta=1.0, code_weights=None, with_corner=True,
                                       corner_class=0, w_corner=1.0))
    for k in ("loss_rcnn_cls", "loss_rcnn_bbox", "loss_rcnn_corner"):
        assert abs(float(ref[k]) - float(mine[k])) < 1e-12, k
    ga = torch.autograd.grad(sum(ref[k] for k in ("loss_rcnn_cls", "loss_rcnn_bbox", "loss_rcnn_corner")), (cls, pred))
    gb = torch.autograd.grad(sum(mine[k] for k in ("loss_rcnn_cls", "loss_rcnn_bbox", "loss_rcnn_corner")), (cls, pred))
    for a, b in zip(ga, gb):
        assert (a - b).abs().max().item() < 1e-12


@pytest.mark.parametrize("rcnn_score_nms", [False, True])
def test_get_bboxes_match_reference(rcnn_score_nms):
    N = RR.load_roi_head()
    test_cfg = dict(use_rotate_nms=True, nms_pre=-1, nms_thr=0.25, score_thr=0.1, min_bbox_size=0, max_num=500,
                    rcnn_score_nms=rcnn_score_nms)
    head = N.build_head(MG.small_head(), None, test_cfg)
    p, l, _, _ = MG.batch([(300, 40)], seed=8)[0]
    g = torch.Generator().manual_seed(1)
    rois = torch.cat([torch.zeros(len(p), 1), p], 1)
    cls, pred = torch.randn(len(p), 1, generator=g) * 2, torch.randn(len(p), 7, generator=g) * 0.2
    valid = torch.rand(len(p), generator=g) > 0.1
    probs = torch.rand(len(p), generator=g)
    out = head.get_bboxes(rois, cls, pred, valid, [l.clone()], [probs.clone()], [dict(box_type_3d=N.Boxes)], cfg=RR.Cfg(test_cfg))[0]
    boxes, scores, labels = RO.get_bboxes(rois, cls, pred, valid, l, probs, 3, 0.1, 0.25, rcnn_score_nms)
    assert torch.equal(out[2], labels)
    assert torch.allclose(out[0].tensor.double(), boxes, atol=1e-5)
    assert torch.allclose(out[1].double(), scores, atol=1e-7)


def test_golden_file_is_the_reference():
    """tests/golden/roi_head_targets.npz holds the reference's fp32 targets of MG.golden_inputs"""
    z = np.load(MG.GOLDEN)
    N = RR.load_roi_head()
    cfg = RR.Cfg(MG.train_cfg())
    out = MG.reference_targets(N, cfg, MG.golden_inputs(seed=7))
    for k, v in out.items():
        assert np.array_equal(z[k], v), k


def test_state_dict_keys_match_reference_for_every_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    from sst_b200.roi_head_modules import FullySparseBboxHead
    N = RR.load_roi_head()
    for rel in CONFIGS:
        m = Config.fromfile(os.path.join(REF_ROOT, "configs", rel))["model"]
        bh = _unshare(dict(m["roi_head"]["bbox_head"]))
        ref = N.build_head(_unshare(bh))
        mine = FullySparseBboxHead(**{k: v for k, v in bh.items() if k != "type"})
        assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, rel
        mine.load_state_dict(ref.state_dict(), strict=True)
        # the heads after the SIR blocks, on the same features
        f = torch.randn(20, sum(sum(c) for c in bh["feat_channels"]), generator=torch.Generator().manual_seed(0))
        ref.eval(), mine.eval()
        with torch.no_grad():
            assert torch.allclose(ref.conv_cls(f), mine.conv_cls(f), atol=1e-6), rel
            assert torch.allclose(ref.conv_reg(f), mine.conv_reg(f), atol=1e-6), rel


def _unshare(x):
    """mmcv's ConfigDict rebuilds every nested list, so `[[16, 32]] * 6` in a config gives six lists; the reference's SIRLayer appends
    to its rel_mlp_hidden_dims in place, so a shared list would grow from block to block"""
    if isinstance(x, dict):
        return {k: _unshare(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_unshare(v) for v in x)
    return x


# settings no config uses but the native sampler accepts, each pinned here so that the GPU edge tests may use the oracle for them:
# (assigners (pos, neg, min_pos) per class, fractions, thresholds, pos_fraction)
SETTINGS = {
    "ignore_band": ([(0.6, 0.3, 0.6), (0.5, 0.2, 0.5), (0.5, 0.25, 0.5)], [0.8, 0.2], [0.55, 0.1], 0.55),
    "min_pos_below_pos": ([(0.7, 0.7, 0.2), (0.6, 0.6, 0.1), (0.6, 0.4, 0.3)], [0.8, 0.2], [0.55, 0.1], 0.55),
    "min_pos_zero": ([(0.45, 0.45, 0.0), (0.35, 0.35, 0.0), (0.35, 0.35, 0.0)], [0.8, 0.2], [0.55, 0.1], 0.55),
    "one_piece": ([(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)], [1.0], [0.55], 0.3),
    "three_pieces": ([(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)], [0.5, 0.3, 0.2], [0.55, 0.3, 0.05], 0.25),
    "pos_fraction_0": ([(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)], [0.8, 0.2], [0.55, 0.1], 0.0),
    "pos_fraction_1": ([(0.45, 0.45, 0.45), (0.35, 0.35, 0.35), (0.35, 0.35, 0.35)], [0.8, 0.2], [0.55, 0.1], 1.0),
}


def _settings_batch(assigners, thrs, per_class, seed, duplicates):
    """four samples as MG.batch draws them, kept 1e-4 away from every threshold of the setting; with duplicates, GT and proposal rows
    repeated so that the argmax, the low-quality match and gt_max_assign_all meet exact ties"""
    t = sorted({v for a in assigners for v in a} | set(thrs))
    out = []
    for b, (n, g) in enumerate([(300, 60), (120, 40), (200, 50), (80, 0)]):
        s = seed * 100 + b
        while True:
            p, l, gt, gl = RO.synth_sample(s, n, g)
            if duplicates and g:
                gt, gl = torch.cat([gt, gt[:g // 3]]), torch.cat([gl, gl[:g // 3]])
                p, l = torch.cat([p, p[: n // 4]]), torch.cat([l, l[: n // 4]])
            if not RO.near_threshold(p, l, gt, gl, [v for v in t if v > 0], per_class=per_class):
                break
            s += 1000
        out.append((p, l, gt, gl))
    return out


@pytest.mark.parametrize("per_class", [True, False])
@pytest.mark.parametrize("setting", list(SETTINGS) + ["duplicates"])
def test_assign_and_sample_settings_match_reference(setting, per_class):
    N = RR.load_roi_head()
    assigners, fr, th, pf = SETTINGS.get(setting, SETTINGS["min_pos_below_pos"])
    if not per_class:
        assigners = assigners[:1]
    num = 96
    a = [dict(type='MaxIoUAssigner', iou_calculator=dict(type='BboxOverlaps3D', coordinate='lidar'), pos_iou_thr=p, neg_iou_thr=n,
              min_pos_iou=m, ignore_iof_thr=-1) for p, n, m in assigners]
    cfg = dict(MG.train_cfg(per_class=per_class, num=num), assigner=a if per_class else a[0],
               sampler=dict(type='IoUNegPiecewiseSampler', num=num, pos_fraction=pf, neg_piece_fractions=fr, neg_iou_piece_thrs=th,
                            neg_pos_ub=-1, add_gt_as_proposals=False, return_iou=True))
    batch = _settings_batch(assigners, th, per_class, 5 + len(setting), setting == "duplicates")
    keys = [torch.rand(len(p), generator=torch.Generator().manual_seed(20 + b), dtype=torch.float64) for b, (p, _, _, _) in enumerate(batch)]
    props = [(N.Boxes(p.double()), torch.rand(len(p)), l) for p, l, _, _ in batch]
    res = N.assign_and_sample(cfg, props, [N.Boxes(g.double()) for _, _, g, _ in batch], [l for _, _, _, l in batch], keys)
    for b, ((p, l, g, gl), r) in enumerate(zip(batch, res)):
        inds, iou, rows, lab, npos = RO.assign_and_sample(p, l, keys[b], g, gl, assigners, per_class, num, pf, fr, th)
        assert torch.equal(inds, torch.cat([r.pos_inds, r.neg_inds])), b
        assert npos == len(r.pos_inds) and len(inds) <= num
        assert torch.equal(rows[:npos], r.pos_assigned_gt_inds)
        assert torch.equal(lab[:npos], r.pos_gt_labels)
        assert torch.equal(iou, r.iou)
