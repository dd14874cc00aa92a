"""CPU: oracle/fsdv2_head_oracle.py against the reference's own FSDV2Head (fsd_v2_head.py over sparse_cluster_head.py and
base_point_bbox_coder.py, imported unmodified through oracle/fsdv2_head_ref.py): labels identical, bbox targets within one ulp, velocity
weights equal and losses (loss_vel included) within 1e-12 in float64, on nuScenes-shaped data (two 5-class tasks, 9- and 10-column GTs,
centroid assignment) and with the tasks' class order permuted against class_names; get_bboxes equal with and without
all_task_max_num.  Also the golden file's contents, the config dicts the GPU tests restate, and for every configs/fsdv2 file the
head's state-dict keys and shapes (strict load) and forward equal to the reference head's."""
import os

import numpy as np
import pytest
import torch

from oracle import cluster_head_oracle as CO
from oracle import fsdv2_head_oracle as FO
from oracle import fsdv2_head_ref as FR
from oracle import make_golden_fsdv2_head as MG

pytestmark = pytest.mark.skipif(not FR.available(), reason="reference tree not present")

CONFIGS = ["fsdv2_waymo_1x.py", "fsdv2_waymo_2x.py", "fsdv2_nusc_1x.py", "fsdv2_nusc_2x.py", "fsdv2_argo_2x.py"]
# a permutation of the nuScenes classes across and within the two tasks
PERM_TASKS = [['pedestrian', 'car', 'barrier', 'truck', 'bicycle'], ['bus', 'traffic_cone', 'motorcycle', 'construction_vehicle', 'trailer']]


def _ulp(a, b):
    nan = a.isnan()
    assert torch.equal(nan, b.isnan())
    return (a[~nan].view(torch.int32).long() - b[~nan].view(torch.int32).long()).abs().max().item() if (~nan).any() else 0


def _head_cfg(tasks=FO.NUSC_TASKS, mode="nusc_l1"):
    m = FO.LOSS_MODES[mode]
    reg = dict(type="SmoothL1Loss", beta=m["beta"]) if m["smooth_l1"] else dict(type="L1Loss")
    return dict(FO.NUSC_HEAD, tasks=[dict(class_names=t) for t in tasks], in_channel=16, shared_mlp_dims=[32],
                loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=m["gamma"], alpha=m["alpha"], loss_weight=m["loss_weight_cls"]),
                loss_center=dict(reg, loss_weight=m["loss_weight_center"]), loss_size=dict(reg, loss_weight=m["loss_weight_size"]),
                loss_rot=dict(reg, loss_weight=m["loss_weight_rot"]), loss_vel=dict(reg, loss_weight=m["loss_weight_vel"]))


@pytest.mark.parametrize("width", [9, 10])
@pytest.mark.parametrize("mode", list(FO.LOSS_MODES))
@pytest.mark.parametrize("order", ["config", "permuted"])
def test_targets_and_losses_match_reference(width, mode, order):
    R = FR.load_fsdv2_head()
    tasks = FO.NUSC_TASKS if order == "config" else PERM_TASKS
    head = FR.build_fsdv2_head(_head_cfg(tasks, mode), FO.NUSC_TRAIN_CFG, FO.NUSC_TEST_CFG)
    xyz, aux, inds, B, L = FO.synth_clusters(7 + width, [500, 0, 400], [30, 5, 25], width=width)
    lab, tg, npos = FO.targets(xyz, inds[:, 1], B, L, tasks, FO.NUSC_NAMES, assign_xyz=aux, code_size=10)
    M = xyz.shape[0]
    x, r = FO.synth_preds(3, M, tasks)
    xd, rd = [a.double() for a in x], [a.double() for a in r]
    ref_losses = head.loss(xd, rd, xyz, inds, [R.Boxes(b) for b in B], L, aux_xyz=aux)
    ref_t = []
    for t in range(len(tasks)):
        gb, gl = head.modify_gt_for_single_task([R.Boxes(b) for b in B], L, t)
        rl, _, rt, rw, _ = head.get_targets(len(tasks[t]), xyz, inds[:, 1], gb, gl, aux_xyz=aux)
        assert torch.equal(rl, lab[t]), t
        assert _ulp(tg[t][:, :10], rt) <= 1
        pos = (rl >= 0) & (rl < len(tasks[t]))
        assert torch.equal(tg[t][pos][:, 8:10], rt[pos][:, 8:10])           # velocity: copied exactly
        assert torch.equal(rw[:, 8], torch.where(pos, tg[t][:, 10], torch.zeros(M))) and torch.equal(rw[:, 8], rw[:, 9])
        assert int(npos[t]) == int(pos.sum())
        ref_t.append(torch.cat([rt, rw[:, 8:9]], 1))
    if width == 10:
        assert any((t[:, 10] == 0).any() and (t[:, 10] == 1).any() for t in tg)   # pasted and genuine positives both present
    # the loss formulas on the reference's own targets (the oracle's sin / cos may be one ulp off torch's CPU ones)
    mine = FO.losses(xd, rd, lab, ref_t, npos, [float(M)] * len(tasks), npos.double(), **FO.LOSS_MODES[mode])
    keys = ("loss_cls", "loss_center", "loss_size", "loss_rot", "loss_vel")
    assert set(ref_losses) == {f"{k}.task{t}" for t in range(len(tasks)) for k in keys}
    for t in range(len(tasks)):
        for q, k in enumerate(keys):
            a, b = float(mine[t, q]), float(ref_losses[f"{k}.task{t}"])
            assert abs(a - b) <= 1e-12 * max(1.0, abs(b)), (t, k, a, b)


def test_centroid_assignment_decides_hits():
    """the in-box test runs on the centroid: some clusters change label against the test on the voxel centre"""
    xyz, aux, inds, B, L = FO.synth_clusters(11, [600, 500], [30, 25])
    a = FO.targets(xyz, inds[:, 1], B, L, FO.NUSC_TASKS, FO.NUSC_NAMES, assign_xyz=aux, code_size=10)[0]
    b = FO.targets(xyz, inds[:, 1], B, L, FO.NUSC_TASKS, FO.NUSC_NAMES, assign_xyz=None, code_size=10)[0]
    assert any(torch.any(u != v) for u, v in zip(a, b))


def test_waymo_code8_and_argo_centroid_match_reference():
    """code size 8: Waymo's head (centre assignment) and Argoverse 2's (centroid assignment), through the same reference head"""
    R = FR.load_fsdv2_head()
    for names, tasks, train_cfg in ((CO.WAYMO_NAMES, CO.WAYMO_TASKS, FO.WAYMO_TRAIN_CFG),
                                    (CO.ARGO_NAMES, CO.ARGO_TASKS, dict(FO.WAYMO_TRAIN_CFG, centroid_assign=True))):
        cfg = dict(FO.WAYMO_HEAD, num_classes=len(names), class_names=names, tasks=[dict(class_names=t) for t in tasks], in_channel=8,
                   shared_mlp_dims=[8])
        head = FR.build_fsdv2_head(cfg, train_cfg)
        xyz, aux, inds, B, L = FO.synth_clusters(5, [400, 300], [25, 20], names, width=9)
        B = [b[:, :7].contiguous() for b in B]
        assign = aux if train_cfg.get("centroid_assign") else None
        lab, tg, npos = FO.targets(xyz, inds[:, 1], B, L, tasks, names, assign_xyz=assign, code_size=8)
        for t in range(len(tasks)):
            gb, gl = head.modify_gt_for_single_task([R.Boxes(b) for b in B], L, t)
            rl, _, rt, _, _ = head.get_targets(len(tasks[t]), xyz, inds[:, 1], gb, gl, aux_xyz=aux)
            assert torch.equal(rl, lab[t]) and _ulp(tg[t], rt) <= 1


@pytest.mark.parametrize("topk", [None, 300])
def test_get_bboxes_match_reference(topk):
    R = FR.load_fsdv2_head()
    test_cfg = dict(FO.NUSC_TEST_CFG, all_task_max_num=topk)
    if topk is None:
        test_cfg.pop("all_task_max_num")
    head = FR.build_fsdv2_head(_head_cfg(PERM_TASKS), FO.NUSC_TRAIN_CFG, test_cfg).eval()
    xyz, _, inds, B, L = FO.synth_clusters(9, [600, 300], [40, 20], spread=15.0)
    M = xyz.shape[0]
    _, r = FO.synth_preds(4, M, PERM_TASKS)
    r = [v * 0.3 for v in r]
    n = M * 10                                  # distinct scores: topk's and the NMS sort's tie orders are their own
    p = torch.linspace(0.02, 0.98, n)[torch.randperm(n, generator=torch.Generator().manual_seed(4))]
    x = [torch.logit(q).reshape(M, 5) for q in p.split(M * 5)]
    got = head.get_bboxes(x, r, xyz, inds, [dict(box_type_3d=R.Boxes)] * 2)
    ref = FO.get_bboxes(x, r, xyz, inds[:, 1], 2, PERM_TASKS, FO.NUSC_NAMES, test_cfg, topk)
    for (a, s, l), (ra, rs, rl) in zip(got, ref):
        assert torch.equal(a.tensor, ra) and torch.equal(s, rs) and torch.equal(l, rl)
        assert ra.shape[1] == 9
    if topk is not None:
        assert ref[0][0].shape[0] == topk
        assert FO.get_bboxes(x, r, xyz, inds[:, 1], 2, PERM_TASKS, FO.NUSC_NAMES, test_cfg)[0][0].shape[0] > topk


def test_golden_file_is_the_reference():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "fsdv2_head_targets.npz"))
    fresh = MG.compute()
    assert set(g.files) == set(fresh)
    for k in g.files:
        assert np.array_equal(g[k], fresh[k], equal_nan=True), k


def test_state_dict_keys_match_reference_for_every_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    from sst_b200.registry import MODELS
    for rel in CONFIGS:
        m = Config.fromfile(os.path.join(REF_ROOT, "configs", "fsdv2", rel))["model"]
        cfg = dict(m["bbox_head"])
        ref = FR.build_fsdv2_head(cfg, m.get("train_cfg"), m.get("test_cfg"))
        mine = MODELS.build(dict(cfg, train_cfg=m.get("train_cfg"), test_cfg=m.get("test_cfg")))
        assert type(mine).__name__ == "FSDV2Head", rel
        assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, rel
        mine.load_state_dict(ref.state_dict(), strict=True)
        feats = torch.randn((50, cfg["in_channel"]), generator=torch.Generator().manual_seed(0))
        ref.eval(), mine.eval()
        with torch.no_grad():
            a, b = ref.forward(feats), mine.forward(feats)
        for k in ("cls_logits", "reg_preds"):
            for u, v in zip(a[k], b[k]):
                assert u.shape == v.shape and torch.allclose(u, v, rtol=1e-6, atol=1e-6), rel
        assert mine.sync_reg_avg_factor == ref.sync_reg_avg_factor and mine.sync_cls_avg_factor == ref.sync_cls_avg_factor, rel


def test_restated_dicts_are_the_configs():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    n = Config.fromfile(os.path.join(REF_ROOT, "configs", "fsdv2", "fsdv2_nusc_1x.py"))["model"]
    assert _plain(n["bbox_head"]) == _plain(FO.NUSC_HEAD)
    assert _plain(n["train_cfg"]) == _plain(FO.NUSC_TRAIN_CFG) and _plain(n["test_cfg"]) == _plain(FO.NUSC_TEST_CFG)
    w = Config.fromfile(os.path.join(REF_ROOT, "configs", "fsdv2", "fsdv2_waymo_1x.py"))["model"]
    assert _plain(w["bbox_head"]) == _plain(FO.WAYMO_HEAD)
    assert _plain(w["train_cfg"]["rpn"]) == _plain(FO.WAYMO_RPN_CFG)
    assert {k: _plain(w["train_cfg"][k]) for k in FO.WAYMO_TRAIN_CFG} == _plain(FO.WAYMO_TRAIN_CFG)


def test_modify_gt_for_single_task_matches_reference_in_any_class_order():
    from sst_b200.registry import MODELS
    R = FR.load_fsdv2_head()
    cfg = dict(_head_cfg(PERM_TASKS), in_channel=8, shared_mlp_dims=[8])
    ref, mine = FR.build_fsdv2_head(cfg), MODELS.build(cfg)
    _, _, _, B, L = FO.synth_clusters(3, [10, 10, 10], [30, 0, 12], width=10)
    boxes = [R.Boxes(b) for b in B]
    for t in range(2):
        rb, rl = ref.modify_gt_for_single_task(boxes, L, t)
        mb, ml = mine.modify_gt_for_single_task(boxes, L, t)
        for a, b, u, v in zip(mb, rb, ml, rl):
            assert type(a) is type(b) and torch.equal(a.tensor, b.tensor) and torch.equal(u, v)


def test_refusals():
    from sst_b200.fsdv2_head_modules import FSDV2Head
    base = dict(FO.NUSC_HEAD, in_channel=8, shared_mlp_dims=[8])
    base.pop("type")
    FSDV2Head(**base)
    for kw in (dict(loss_iou=dict(type="CrossEntropyLoss")), dict(iou_mlp=[64]), dict(corner_loss_cfg=dict(delta=1.0)),
               dict(enlarge_width=0.1), dict(loss_vel=None), dict(loss_vel=dict(type="SmoothL1Loss", beta=0.1)),
               dict(bbox_coder=dict(type="BasePointBBoxCoder", code_size=9)),
               dict(common_attrs=dict(center=(3, 2, 8), dim=(3, 2, 8), rot=(2, 2, 8))),
               dict(tasks=[dict(class_names=FO.NUSC_NAMES[:5]), dict(class_names=FO.NUSC_NAMES[4:9])])):
        with pytest.raises(ValueError):
            FSDV2Head(**dict(base, **kw))
    h = FSDV2Head(**base)
    for cfg in (dict(assign_by_dist=True), dict(max_assign_dist=2.0), dict(code_weight=[1.0] * 10)):
        with pytest.raises(ValueError):
            h.train_cfg = cfg
    h.test_cfg = dict(FO.NUSC_TEST_CFG, nms_pre=100)
    with pytest.raises(ValueError):
        h.get_bboxes([torch.zeros(1, 5)] * 2, [torch.zeros(1, 10)] * 2, torch.zeros(1, 3), torch.zeros(1, dtype=torch.long), [dict()])
    h.test_cfg = dict(FO.NUSC_TEST_CFG, nms_thr=[0.2] * 5)
    with pytest.raises(ValueError):
        h.get_bboxes([torch.zeros(1, 5)] * 2, [torch.zeros(1, 10)] * 2, torch.zeros(1, 3), torch.zeros(1, dtype=torch.long), [dict()])


def _plain(d):
    if isinstance(d, dict):
        return {k: _plain(v) for k, v in d.items()}
    if isinstance(d, (list, tuple)):
        return [_plain(v) for v in d]
    return d
