"""CPU: oracle/cluster_head_oracle.py against the reference's own SparseClusterHeadV2 (sparse_cluster_head{,_v2}.py and
base_point_bbox_coder.py, imported unmodified through oracle/cluster_head_ref.py): labels identical, bbox targets within one ulp (the
oracle rounds its log / sin / cos from float64, torch's CPU kernels are within an ulp of that), losses within 1e-12 in float64, get_bboxes
equal for the training `rpn` cfg (no NMS) and the test cfg (rotated NMS), on Waymo's three single-class tasks and on Argoverse 2's six
multi-class groups with boxes overlapping across classes.  Also the golden file's contents, and for every config that declares the head,
state-dict keys and shapes equal to the reference head's."""
import os

import numpy as np
import pytest
import torch

from oracle import cluster_head_oracle as CO
from oracle import cluster_head_ref as CR
from oracle import make_golden_cluster_head as MG

pytestmark = pytest.mark.skipif(not CR.available(), reason="reference tree not present")

CONFIGS = ["fsd/fsd_waymoD1_1x.py", "fsd/fsd_waymoD1_1x_3f.py", "fsd/fsd_waymoD1_1x_sst_encoder.py", "fsd/fsd_waymoD1_1x_submission.py",
           "fsdpp/fsdpp_waymoD1_1x_7f_6base.py", "argo2/argo_onestage_12e.py"]


def _head(names, tasks, loss_mode="fsd_l1"):
    m = CO.LOSS_MODES[loss_mode]
    reg = dict(type="SmoothL1Loss", beta=m["beta"]) if m["smooth_l1"] else dict(type="L1Loss")
    cfg = dict(CO.FSD_D1_HEAD, num_classes=len(names), class_names=names, tasks=[dict(class_names=t) for t in tasks], in_channel=16,
               shared_mlp_dims=[32], loss_cls=dict(type="FocalLoss", use_sigmoid=True, gamma=m["gamma"], alpha=m["alpha"],
                                                   loss_weight=m["loss_weight_cls"]),
               loss_center=dict(reg, loss_weight=m["loss_weight_center"]), loss_size=dict(reg, loss_weight=m["loss_weight_size"]),
               loss_rot=dict(reg, loss_weight=m["loss_weight_rot"]))
    return CR.build_cluster_head(cfg, CO.FSD_D1_TRAIN_CFG, CO.FSD_D1_TEST_CFG)


def _ulp(a, b):
    nan = a.isnan()
    assert torch.equal(nan, b.isnan())
    return (a[~nan].view(torch.int32).long() - b[~nan].view(torch.int32).long()).abs().max().item() if (~nan).any() else 0


CASES = {"waymo": (CO.WAYMO_NAMES, CO.WAYMO_TASKS, "fsd_l1"), "argo": (CO.ARGO_NAMES, CO.ARGO_TASKS, "argo_smoothl1")}


@pytest.mark.parametrize("case", list(CASES))
def test_targets_and_losses_match_reference(case):
    names, tasks, mode = CASES[case]
    R = CR.load_cluster_head()
    head = _head(names, tasks, mode)
    xyz, inds, B, L = CO.synth_clusters(7, [500, 0, 400], [30, 5, 25], names)
    for b in (0, 2):                          # a second box of another class on top of each of the first boxes
        B[b][1::2] = B[b][0:-1:2]
    lab, tg, npos = CO.targets(xyz, inds[:, 1], B, L, tasks, names)
    M = xyz.shape[0]
    x, r = CO.synth_preds(3, M, tasks)
    xd, rd = [a.double() for a in x], [a.double() for a in r]
    ref_losses = head.loss(xd, rd, xyz, inds, [R.Boxes(b) for b in B], L)
    ref_t = []
    for t in range(len(tasks)):
        gb, gl = head.modify_gt_for_single_task([R.Boxes(b) for b in B], L, t)
        rl, _, rt, _, _ = head.get_targets(len(tasks[t]), xyz, inds[:, 1], gb, gl)
        assert torch.equal(rl, lab[t]), t
        assert _ulp(tg[t], rt) <= 1
        assert int(npos[t]) == int(((rl >= 0) & (rl < len(tasks[t]))).sum())
        ref_t.append(rt)
    # the loss formulas on the reference's own targets (the oracle's sin / cos may be one ulp off torch's CPU ones)
    mine = CO.losses(xd, rd, lab, ref_t, npos, [float(M)] * len(tasks), npos.double(), **CO.LOSS_MODES[mode])
    for t in range(len(tasks)):
        for q, k in enumerate(("loss_cls", "loss_center", "loss_size", "loss_rot")):
            a, b = float(mine[t, q]), float(ref_losses[f"{k}.task{t}"])
            assert abs(a - b) <= 1e-12 * max(1.0, abs(b)), (t, k, a, b)
    if case == "argo":                        # the rank order decided some hits: a lower-index box of a later class held the cluster
        assert any(torch.any(a != b) for a, b in zip(lab, CO.targets(xyz, inds[:, 1], B, L, [t[::-1] for t in tasks], names)[0]))


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("cfg", ["rpn", "test"])
def test_get_bboxes_match_reference(case, cfg):
    names, tasks, _ = CASES[case]
    R = CR.load_cluster_head()
    head = _head(names, tasks)
    head.train(cfg == "rpn")
    xyz, inds, B, L = CO.synth_clusters(9, [600, 300], [40, 20], names, spread=15.0)
    x, r = CO.synth_preds(4, xyz.shape[0], tasks)
    r = [v * 0.3 for v in r]
    got = head.get_bboxes(x, r, xyz, inds, [dict(box_type_3d=R.Boxes)] * 2)
    ref = CO.get_bboxes(x, r, xyz, inds[:, 1], 2, tasks, names, CO.RPN_CFG if cfg == "rpn" else CO.TEST_CFG)
    for (a, s, l), (ra, rs, rl) in zip(got, ref):
        assert torch.equal(a.tensor, ra) and torch.equal(s, rs) and torch.equal(l, rl)


def test_get_bboxes_batch_of_one_keeps_every_cluster():
    """eval mode, B = 1: the reference's split_by_batch returns every cluster, out-of-range batch index or not; the oracle follows"""
    R = CR.load_cluster_head()
    head = _head(CO.WAYMO_NAMES, CO.WAYMO_TASKS)
    head.eval()
    xyz, inds, B, L = CO.synth_clusters(5, [400], [20], CO.WAYMO_NAMES)
    inds[3, 1], inds[9, 1] = 4, -1
    x, r = CO.synth_preds(6, xyz.shape[0], CO.WAYMO_TASKS)
    got = head.get_bboxes(x, r, xyz, inds, [dict(box_type_3d=R.Boxes)])
    ref = CO.get_bboxes(x, r, xyz, inds[:, 1], 1, CO.WAYMO_TASKS, CO.WAYMO_NAMES, CO.TEST_CFG)
    (a, s, l), (ra, rs, rl) = got[0], ref[0]
    assert torch.equal(a.tensor, ra) and torch.equal(s, rs) and torch.equal(l, rl)


def test_modify_gt_for_single_task_matches_reference():
    """the module's modify_gt_for_single_task (torch only, so it runs on the CPU) gives the reference's box objects and labels"""
    from sst_b200.registry import MODELS
    R = CR.load_cluster_head()
    names, tasks = CO.ARGO_NAMES, CO.ARGO_TASKS
    cfg = dict(CO.FSD_D1_HEAD, num_classes=len(names), class_names=names, tasks=[dict(class_names=t) for t in tasks], in_channel=8,
               shared_mlp_dims=[8])
    ref, mine = CR.build_cluster_head(cfg), MODELS.build(cfg)
    _, _, B, L = CO.synth_clusters(3, [10, 10, 10], [30, 0, 12], names)
    boxes = [R.Boxes(b) for b in B]
    for t in range(len(tasks)):
        rb, rl = ref.modify_gt_for_single_task(boxes, L, t)
        mb, ml = mine.modify_gt_for_single_task(boxes, L, t)
        for a, b, u, v in zip(mb, rb, ml, rl):
            assert type(a) is type(b) and torch.equal(a.tensor, b.tensor) and torch.equal(u, v)


def test_golden_file_is_the_reference():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "cluster_head_targets.npz"))
    fresh = MG.compute()
    assert set(g.files) == set(fresh)
    for k in g.files:
        assert np.array_equal(g[k], fresh[k], equal_nan=True), k


def test_state_dict_keys_match_reference_for_every_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    from sst_b200.registry import MODELS
    for rel in CONFIGS:
        m = Config.fromfile(os.path.join(REF_ROOT, "configs", rel))["model"]
        cfg = dict(m["bbox_head"])
        ref = CR.build_cluster_head(cfg, m.get("train_cfg"), m.get("test_cfg"))
        mine = MODELS.build(dict(cfg, train_cfg=m.get("train_cfg"), test_cfg=m.get("test_cfg")))
        assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, rel
        mine.load_state_dict(ref.state_dict())
        feats = torch.randn((50, cfg["in_channel"]), generator=torch.Generator().manual_seed(0))
        ref.eval(), mine.eval()
        with torch.no_grad():
            a, b = ref.forward(feats), mine.forward(feats)
        for k in ("cls_logits", "reg_preds"):
            for u, v in zip(a[k], b[k]):
                assert torch.allclose(u, v, rtol=1e-6, atol=1e-6), rel
        assert mine.sync_reg_avg_factor == ref.sync_reg_avg_factor and mine.sync_cls_avg_factor == ref.sync_cls_avg_factor, rel


def test_training_head_dict_is_the_config():
    from oracle.ref_shim import REF_ROOT
    from sst_b200.config import Config
    m = Config.fromfile(os.path.join(REF_ROOT, "configs", "fsd", "fsd_waymoD1_1x.py"))["model"]
    assert _plain(m["bbox_head"]) == _plain(CO.FSD_D1_HEAD)
    assert _plain(m["train_cfg"]["rpn"]) == _plain(CO.RPN_CFG) and _plain(m["test_cfg"]["rpn"]) == _plain(CO.TEST_CFG)


def _plain(d):
    if isinstance(d, dict):
        return {k: _plain(v) for k, v in d.items()}
    if isinstance(d, (list, tuple)):
        return [_plain(v) for v in d]
    return d
