"""CPU: oracle/anchor3d_oracle.py against the reference's own Anchor3DHead (anchor3d_head.py, train_mixins.py and the reference's anchor
generator, box coder, IoU calculator and box3d_multiclass_nms, imported unmodified through oracle/anchor3d_ref.py): targets bit-identical,
float64 losses and gradients within 1e-12 relative, get_bboxes equal; and sst_b200's SECONDFPN / Anchor3DHead with the reference's
state-dict keys and shapes for every configs/sst* file that uses them."""
import glob
import os

import pytest
import torch

from oracle import anchor3d_oracle as AO
from oracle import anchor3d_ref as AR

pytestmark = pytest.mark.skipif(not AR.available(), reason="reference tree not present")

CASES = [("default", {}, [40, 0, 25]), ("per_class", dict(assign_per_class=True), [30, 12]),
         ("argmax_only", dict(gt_max_assign_all=False), [50]), ("min_pos_0", dict(thresholds=[(0.5, 0.3, 0.0)] * 3), [20, 3]),
         ("nonsquare", dict(height=20, width=70, classes=(1, 2)), [35]), ("one_col", dict(height=40, width=1), [6, 0])]


def _ref_targets(geom, head, boxes, labels):
    R = AR.load_anchor_head()
    metas = [{}] * len(boxes)
    anchors = head.get_anchors([(geom["H"], geom["W"])], metas, device="cpu")
    return head.anchor_target_3d(anchors, [R.Boxes(b) for b in boxes], metas, gt_labels_list=labels,
                                 num_classes=geom["head"]["num_classes"], label_channels=1, sampling=False)


@pytest.mark.parametrize("name,kw,sizes", CASES, ids=[c[0] for c in CASES])
def test_oracle_targets_bit_identical_to_reference(name, kw, sizes):
    geom = AO.geometry(**kw)
    head = AR.build_anchor_head(geom)
    boxes, labels = AO.synth_batch(sum(map(ord, name)), geom, sizes)
    ref = _ref_targets(geom, head, boxes, labels)
    anchors = AO.anchors_from_axes(*AO.axes(geom))
    assert torch.equal(head.get_anchors([(geom["H"], geom["W"])], [{}], device="cpu")[0][0].reshape(-1, 7), anchors.reshape(-1, 7))
    got = AO.targets(anchors, boxes, labels, AO.assigner_args(geom), geom["head"]["num_classes"], geom["head"]["assign_per_class"],
                     geom["head"]["dir_offset"])
    for k in range(6):
        assert torch.equal(ref[k][0], got[k]), f"output {k} differs"
    assert ref[6] == got[6]
    assert (got[0] < geom["head"]["num_classes"]).any()


def test_sst_b200_generator_axes_match_reference():
    from sst_b200.anchor3d_modules import AlignedAnchor3DRangeGenerator
    for kw in ({}, dict(height=1, width=33), dict(height=468, width=468)):
        geom = AO.geometry(**kw)
        R = AR.load_anchor_head()
        g = dict(geom["head"]["anchor_generator"])
        g.pop("type")
        ref = R.AlignedAnchor3DRangeGenerator(**g).grid_anchors([(geom["H"], geom["W"])], device="cpu")[0]
        mine = AlignedAnchor3DRangeGenerator(**g).grid_anchors([(geom["H"], geom["W"])], device="cpu")[0]
        assert torch.equal(ref, mine)


def test_oracle_losses_match_reference_float64():
    geom = AO.geometry()
    head = AR.build_anchor_head(geom).double()
    boxes, labels = AO.synth_batch(9, geom, [40, 0, 25])
    cls, reg, dr = (x.double() for x in AO.synth_preds(9, geom, 3, 3.0))
    a = [x.clone().requires_grad_(True) for x in (cls, reg, dr)]
    R = AR.load_anchor_head()
    ref = head.loss([a[0]], [a[1]], [a[2]], [R.Boxes(b) for b in boxes], labels, [{}] * 3)
    ref_vals = [ref["loss_cls"][0], ref["loss_bbox"][0], ref["loss_dir"][0]]
    sum(ref_vals).backward()
    t = AO.targets(AO.anchors_from_axes(*AO.axes(geom)), boxes, labels, AO.assigner_args(geom), 3)
    b = [x.clone().requires_grad_(True) for x in (cls, reg, dr)]
    lc = AO.focal_loss(b[0], t[0], t[1], t[6], 3, 1.0)
    lb, ld = AO.reg_dir_loss(b[1], b[2], t[0], t[2], t[3], t[4], t[5], t[6], 3, [1.0] * 7, 0.5, 0.2)
    for r, g in zip(ref_vals, (lc, lb, ld)):
        assert abs(r.item() - g.item()) <= 1e-12 * abs(r.item())
    (lc + lb + ld).backward()
    for x, y in zip(a, b):
        assert (x.grad - y.grad).abs().max() <= 1e-12 * x.grad.abs().max()


def test_oracle_get_bboxes_matches_reference():
    R = AR.load_anchor_head()
    for classes in ((1, 2), (0, 1, 2)):
        geom = AO.geometry(height=50, width=70, classes=classes)
        cfg = dict(geom["test_cfg"], nms_pre=1500)
        head = AR.build_anchor_head(dict(geom, test_cfg=cfg))
        cls, reg, dr = AO.synth_preds(21, geom, 2)
        got = head.get_bboxes([cls], [reg], [dr], [{"box_type_3d": R.Boxes}] * 2)
        anchors = AO.anchors_from_axes(*AO.axes(geom)).reshape(-1, 7)
        for b in range(2):
            mine = AO.get_bboxes_single(cls[b], reg[b], dr[b], anchors, len(classes), cfg)
            assert mine[0].shape[0] > 0
            assert torch.equal(got[b][0].tensor, mine[0]) and torch.equal(got[b][1], mine[1]) and torch.equal(got[b][2], mine[2])


def _configs():
    root = os.path.join(AR.REF_ROOT, "configs")
    return sorted(glob.glob(os.path.join(root, "sst", "*.py")) + glob.glob(os.path.join(root, "sst_refactor", "*.py")))


def test_state_dict_keys_and_shapes_match_reference_for_every_config():
    from sst_b200.config import Config
    from sst_b200.registry import MODELS
    R = AR.load_anchor_head()
    seen = 0
    for path in _configs():
        try:
            m = Config.fromfile(path)["model"]
        except Exception:       # files that do not load as configs (work in progress upstream) use neither module
            continue
        if m.get("neck", {}).get("type") == "SECONDFPN":
            c = dict(m["neck"])
            c.pop("type")
            ref, mine = R.SECONDFPN(**c), MODELS.build(m["neck"])
            assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, path
        if m.get("bbox_head", {}).get("type") == "Anchor3DHead":
            ref = AR.build_anchor_head(m["bbox_head"], m["train_cfg"], m["test_cfg"])
            mine = MODELS.build(dict(m["bbox_head"], train_cfg=m["train_cfg"], test_cfg=m["test_cfg"]))
            assert {k: v.shape for k, v in ref.state_dict().items()} == {k: v.shape for k, v in mine.state_dict().items()}, path
            seen += 1
    assert seen >= 7


def test_flagship_dicts_are_the_config():
    from sst_b200 import flagship as fl
    from sst_b200.config import Config
    m = Config.fromfile(os.path.join(AR.REF_ROOT, "configs/sst_refactor/sst_waymoD5_1x_3class_8heads_v2.py"))["model"]
    assert (m["neck"], m["bbox_head"], m["train_cfg"], m["test_cfg"]) == (fl.ANCHOR_NECK, fl.ANCHOR_HEAD, fl.ANCHOR_TRAIN_CFG,
                                                                          fl.ANCHOR_TEST_CFG)
