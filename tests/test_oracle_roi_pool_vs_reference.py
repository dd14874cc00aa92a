"""CPU, build container only: pins the RoI point-pooling restatement (oracle/roi_pool_oracle.dynamic_point_pool, SURVEY 8f next-3) to the
reference's own box test - points_in_boxes_cpu of mmdet3d/ops/roiaware_pool3d/src, compiled unmodified into oracle/_ref by
oracle/build_ref_roiaware.py.  The original and the enlarged box (x, y, z_bottom - e2/2, w + e0, l + e1, h + e2, rz) must give the same membership,
except for pairs within 1e-4 m of a face (the CPU twin has no fused multiply-add and may round cos / sin differently)."""
import math

import pytest
import torch

from oracle import build_ref, roi_pool_oracle as RO

REF = build_ref.load_module("roiaware_pool3d_ext_ref")
pytestmark = pytest.mark.skipif(REF is None, reason="oracle/_ref roiaware_pool3d build not present")
EXTRA = [0.5, 0.5, 0.5]


def _frame(seed, yaw):
    pts, rois, _, _ = RO.synth_roi_frame(seed, n_pts=20000, n_rois=80, spread=12.0)   # dense: boxes overlap
    g = torch.Generator().manual_seed(seed + 100)
    if yaw == "random":
        rois[:, 6] = (torch.rand(rois.shape[0], generator=g) - 0.5) * 4 * math.pi
    else:
        rois[:, 6] = yaw
    return pts, rois


def _ref_membership(boxes, pts):
    out = torch.zeros((boxes.shape[0], pts.shape[0]), dtype=torch.int32)
    REF.points_in_boxes_cpu(boxes.contiguous(), pts.contiguous(), out)
    return out.bool()


def _face_distance(boxes, pts):
    """float64 distance of every point to the nearest face of every box (negative outside)"""
    b, p = boxes.double(), pts.double()
    cz = b[:, 2] + b[:, 5] / 2
    a = b[:, 6] + math.pi / 2
    sx, sy = p[None, :, 0] - b[:, None, 0], p[None, :, 1] - b[:, None, 1]
    lx = sx * torch.cos(a)[:, None] - sy * torch.sin(a)[:, None]
    ly = sx * torch.sin(a)[:, None] + sy * torch.cos(a)[:, None]
    dz = (p[None, :, 2] - cz[:, None]).abs()
    return torch.stack([b[:, None, 4] / 2 - lx.abs(), b[:, None, 3] / 2 - ly.abs(), b[:, None, 5] / 2 - dz]).abs().amin(0)


@pytest.mark.parametrize("yaw", [0.0, math.pi / 2, -math.pi / 2, math.pi, "random"])
def test_membership_matches_reference_box_test(yaw):
    pts, rois = _frame(3, yaw)
    near_total = 0
    for boxes in (rois, RO.enlarge_boxes(rois, EXTRA)):
        ours, _, _, _ = RO.box_test(pts, boxes)
        ref = _ref_membership(boxes, pts)
        assert ref.sum() > 1000
        diff = ours != ref
        if diff.any():
            assert (_face_distance(boxes, pts)[diff] < 1e-4).all(), "membership differs away from a face"
        near_total += int(diff.sum())
    assert near_total <= 5


@pytest.mark.parametrize("yaw", [0.0, "random"])
def test_pool_rows_follow_membership_and_identities(yaw):
    pts, rois = _frame(7, yaw)
    cap = 40
    idx, roi, feats = RO.dynamic_point_pool(rois, pts, EXTRA, cap)
    big = _ref_membership(RO.enlarge_boxes(rois, EXTRA), pts)
    orig = _ref_membership(rois, pts)
    # rows: per RoI its first `cap` points of the enlarged box in input order, RoIs ascending
    exp_roi, exp_idx = [], []
    for r in range(rois.shape[0]):
        i = big[r].nonzero()[:, 0][:cap]
        exp_idx.append(i)
        exp_roi.append(torch.full_like(i, r))
    exp_idx, exp_roi = torch.cat(exp_idx), torch.cat(exp_roi)
    near = _face_distance(RO.enlarge_boxes(rois, EXTRA), pts)
    if not (torch.equal(idx, exp_idx) and torch.equal(roi, exp_roi)):   # only a face-grazing point may move the cut
        assert (near[big != RO.box_test(pts, RO.enlarge_boxes(rois, EXTRA))[0]] < 1e-4).all()
    else:
        margin = ~orig[roi, idx]
        ok = near[roi, idx] > 1e-4
        assert torch.equal(feats[ok, 12].bool(), margin[ok])
    # the reference extractor's debug asserts (dynamic_point_roi_extractor.py:92-101)
    r = rois[roi]
    assert torch.equal(feats[:, :3], pts[idx])
    assert torch.isclose(feats[:, 6] + feats[:, 9], r[:, 4]).all()
    assert torch.isclose(feats[:, 7] + feats[:, 10], r[:, 3]).all()
    assert torch.isclose(feats[:, 8] + feats[:, 11], r[:, 5]).all()
    for k, dim in ((0, 4), (1, 3), (2, 5)):
        assert (feats[:, 3 + k].abs() < r[:, dim] + EXTRA[k] + 1e-5).all()
    # margin rows have a negative offset, inner rows none
    inner = feats[:, 12] == 0
    assert (feats[inner, 6:12] >= -1e-5).all() and (feats[~inner, 6:12].amin(1) < 1e-5).all()


def test_fake_row_and_capacity():
    pts, rois = _frame(5, "random")
    far = rois.clone()
    far[:, 0] += 1000.0
    idx, roi, feats = RO.dynamic_point_pool(far, pts, EXTRA, 16)
    assert idx.tolist() == [-1] and roi.tolist() == [-1] and torch.equal(feats, torch.zeros((1, 13)))
    full = RO.dynamic_point_pool(rois, pts, EXTRA, 16)
    cut = RO.dynamic_point_pool(rois, pts, EXTRA, 16, max_all_pts=100)
    assert full[0].numel() > 100 and all(torch.equal(a[:100], b) for a, b in zip(full, cut))
