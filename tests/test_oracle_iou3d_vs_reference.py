"""CPU: pins the rotated BEV IoU / NMS restatement (oracle/iou3d_oracle.py) - its overlap areas against an independent exact computation
(scipy HalfspaceIntersection + ConvexHull in float64), its IoU and keep lists against the reference's own CUDA kernels through the golden
fixture tests/golden/iou3d_bev.npz (written on a GPU by oracle/make_golden_iou3d.py), and its box3d_multiclass_nms against the
reference's own function, run unmodified where the reference tree exists."""
import math
import os
import types

import numpy as np
import pytest
import torch

from oracle import iou3d_oracle as IO, ref_shim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "iou3d_bev.npz")


def _halfspaces(box):
    """the rectangle as 4 half-spaces A x + b <= 0 (scipy's layout), from its corners"""
    c = IO.corners(box)[0]
    if (box[2] - box[0]) * (box[3] - box[1]) < 0:
        c = c[::-1]
    hs = []
    for k in range(4):
        p, q = c[k], c[(k + 1) % 4]
        n = np.array([q[1] - p[1], p[0] - q[0]])          # outward normal of a counter-clockwise edge
        hs.append([n[0], n[1], -n @ p])
    return np.array(hs)


def exact_overlap(a, b):
    from scipy.optimize import linprog
    from scipy.spatial import ConvexHull, HalfspaceIntersection
    if (a[2] - a[0]) * (a[3] - a[1]) == 0 or (b[2] - b[0]) * (b[3] - b[1]) == 0:
        return 0.0
    hs = np.vstack([_halfspaces(a), _halfspaces(b)])
    norm = np.linalg.norm(hs[:, :2], axis=1)
    # Chebyshev centre: the deepest interior point
    res = linprog([0, 0, -1], A_ub=np.hstack([hs[:, :2], norm[:, None]]), b_ub=-hs[:, 2], bounds=[(None, None)] * 2 + [(0, None)])
    if not res.success or res.x[2] < 1e-9:
        return 0.0
    pts = HalfspaceIntersection(hs, res.x[:2]).intersections
    return ConvexHull(pts).volume


def test_overlap_vs_exact_halfspace_intersection():
    sp = IO.special_boxes().double().numpy()
    dense = IO.synth_boxes(41, 160, objects=12).double().numpy()
    pairs = [(sp[i], sp[j]) for i in range(len(sp)) for j in range(len(sp))]
    pairs += [(dense[i], dense[j]) for i in range(0, 160, 2) for j in range(1, 160, 7)]
    a = np.array([p[0] for p in pairs])
    b = np.array([p[1] for p in pairs])
    got = IO.overlap_pairs(a, b)
    exact = np.array([exact_overlap(x, y) for x, y in pairs])
    assert (exact > 0).sum() > 200
    assert np.abs(got - exact).max() <= 1e-9 * max(1.0, exact.max()), np.abs(got - exact).max()


def test_axis_aligned_values():
    b = torch.tensor([[0, 0, 2, 1, 0.0], [1, 0, 3, 1, 0.0], [-0.5, -0.5, 0.5, 0.5, 0.0], [-0.5, -0.5, 0.5, 0.5, math.pi / 4]])
    ov = IO.boxes_overlap_bev(b, b)
    assert ov[0, 1] == 1.0 and abs(IO.boxes_iou_bev(b, b)[0, 1].item() - 1 / 3) < 1e-15
    assert abs(ov[2, 3].item() - 2 * (math.sqrt(2) - 1)) < 1e-12


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_oracle_iou_vs_reference_golden(golden):
    a, b = torch.from_numpy(golden["boxes_a"]), torch.from_numpy(golden["boxes_b"])
    iou, ov = IO.boxes_iou_bev(a, b).numpy(), IO.boxes_overlap_bev(a, b).numpy()
    # the reference returns garbage for zero-area boxes (IoU 3.09 and 30.85 in this fixture); the oracle gives 0 there
    ok = ((golden["boxes_a"][:, 2] - golden["boxes_a"][:, 0]) * (golden["boxes_a"][:, 3] - golden["boxes_a"][:, 1]) != 0)[:, None] & \
         ((golden["boxes_b"][:, 2] - golden["boxes_b"][:, 0]) * (golden["boxes_b"][:, 3] - golden["boxes_b"][:, 1]) != 0)[None, :]
    assert (golden["iou"] > 0).sum() > 1000 and (~ok).sum() > 0
    assert np.abs(iou - golden["iou"])[ok].max() <= 2e-5
    assert (np.abs(ov - golden["overlap"]) / np.maximum(np.abs(ov), 1.0))[ok].max() <= 2e-5
    assert (iou[~ok] == 0).all() and (ov[~ok] == 0).all()


def test_oracle_keep_lists_vs_reference_golden(golden):
    boxes, scores = torch.from_numpy(golden["nms_boxes"]), torch.from_numpy(golden["nms_scores"])
    for t in golden["thresholds"]:
        assert np.array_equal(IO.nms_gpu(boxes, scores, float(t)).numpy(), golden[f"keep_rot_{t}"])
        assert np.array_equal(IO.nms_normal_gpu(boxes, scores, float(t)).numpy(), golden[f"keep_normal_{t}"])


@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present")
def test_multiclass_nms_vs_reference_function():
    ref = ref_shim.reference_functions("mmdet3d/core/post_processing/box3d_nms.py", ["box3d_multiclass_nms"],
                                       extra_globals={"nms_gpu": IO.nms_gpu, "nms_normal_gpu": IO.nms_normal_gpu})["box3d_multiclass_nms"]
    g = torch.Generator().manual_seed(5)
    n = 600
    bfn = IO.synth_boxes(43, n, objects=60)
    bboxes = torch.rand(n, 7, generator=g)
    scores = (torch.randperm(n * 4, generator=g).double() / (n * 4)).float().view(n, 4)
    dirs, b2d = torch.rand(n, generator=g), torch.rand(n, 4, generator=g)
    for rotate in (True, False):
        for score_thr, nms_thr, max_num, extra in (([0.1, 0.3, 0.2], [0.25, 0.1, 0.5], 500, dict(mlvl_dir_scores=dirs)),
                                                   (0.2, 0.25, 100, dict(mlvl_dir_scores=dirs, mlvl_attr_scores=dirs, mlvl_bboxes2d=b2d)),
                                                   ([0.1, 0.3, 0.2], [0.25, None, 0.7], 10000, {}),
                                                   (2.0, 0.25, 500, dict(mlvl_dir_scores=dirs, mlvl_bboxes2d=b2d))):
            cfg = types.SimpleNamespace(use_rotate_nms=rotate, nms_thr=nms_thr)
            want = ref(bboxes, bfn, scores, score_thr, max_num, cfg, **extra)
            got = IO.box3d_multiclass_nms(bboxes, bfn, scores, score_thr, max_num, cfg, **extra)
            assert len(got) == len(want)
            for x, y in zip(got, want):
                assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y)
