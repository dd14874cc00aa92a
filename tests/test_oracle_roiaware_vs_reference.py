"""CPU: pins the roiaware_pool3d restatement (oracle/roiaware_oracle.py) to the reference.  Membership against the reference's own
points_in_boxes_cpu (compiled unmodified into oracle/_ref by oracle/build_ref_roiaware.py, build container only); points_in_boxes_gpu /
_batch, the RoIAwarePool3d forward (voxel indices, counts, argmax, pooled values: bitwise) and backward (1e-6 relative) against
tests/golden/roiaware_pool3d.npz, written from the reference's CUDA kernels on an H100 by oracle/make_golden_roiaware.py.  Also the
host-side argument checks of ops.RoIAwarePool3d."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import build_ref, roi_pool_oracle as RO, roiaware_oracle as RA

REF = build_ref.load_module("roiaware_pool3d_ext_ref")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "roiaware_pool3d.npz")


@pytest.mark.skipif(REF is None, reason="oracle/_ref roiaware_pool3d build not present")
@pytest.mark.parametrize("yaw", [0.0, -math.pi / 2, "random"])
def test_membership_matches_reference_points_in_boxes_cpu(yaw):
    pts, rois, _, _ = RO.synth_roi_frame(31, n_pts=20000, n_rois=64, spread=12.0)
    if yaw == "random":
        rois[:, 6] = (torch.rand(rois.shape[0], generator=torch.Generator().manual_seed(5)) - 0.5) * 4 * math.pi
    else:
        rois[:, 6] = yaw
    ref = torch.zeros((rois.shape[0], pts.shape[0]), dtype=torch.int32)
    REF.points_in_boxes_cpu(rois.contiguous(), pts.contiguous(), ref)
    ours = RA.points_in_boxes_batch(pts[None], rois[None])[0].t()
    assert ref.sum() > 1000
    assert (ours != ref).sum() <= 3     # the CPU twin has no fused multiply-add: a point within rounding of a face may differ


def test_golden_inputs_cover_the_cases():
    x = RA.golden_inputs()
    _, _, pidx = RA.roiaware_pool3d(x["rois"], x["pts"], x["feats"], x["out_size"], x["m"], 0)
    assert (pidx[..., 0] == x["m"] - 1).any()                            # a voxel holding more points than it keeps
    inside = RA.membership(x["pts"], x["rois"])[0]
    assert (inside.sum(0) > 1).any()                                     # overlapping RoIs
    assert x["out_size"][0] != x["out_size"][1]


def _golden():
    g = np.load(GOLDEN)
    return {k: torch.from_numpy(g[k]) for k in g.files}


def _bits(t):
    """fp32 as its bit patterns (so -0.0 != 0.0), every NaN as one pattern: NaN payloads differ between CPU and GPU arithmetic"""
    t = t.cpu().contiguous()
    if t.dtype != torch.float32:
        return t
    return torch.where(torch.isnan(t), torch.full_like(t, float("nan")), t).view(torch.int32)


@pytest.mark.parametrize("mode", [0, 1])
def test_pool3d_matches_golden(mode):
    g = _golden()
    out_size, m = tuple(g["out_size"].tolist()), int(g["m"])
    pooled, argmax, pidx = RA.roiaware_pool3d(g["rois"], g["pts"], g["feats"], out_size, m, mode)
    assert torch.equal(pidx, g[f"pts_idx_{mode}"])                    # voxel indices, counts, first m - 1 points
    assert torch.equal(_bits(pooled), _bits(g[f"pooled_{mode}"]))      # bitwise, NaN included
    if mode == 0:
        assert torch.equal(argmax, g["argmax_0"])
    grad = RA.roiaware_pool3d_backward(pidx, argmax, g["grad"], g["pts"].shape[0], mode)
    ref = g[f"grad_in_{mode}"]
    assert ref.abs().sum() > 0
    torch.testing.assert_close(grad, ref, rtol=1e-6, atol=1e-6 * ref.abs().max().item())


def test_points_in_boxes_match_golden():
    g = _golden()
    assert torch.equal(RA.points_in_boxes_gpu(g["pib_pts"], g["pib_boxes"]), g["pib_first"])
    assert torch.equal(RA.points_in_boxes_batch(g["pib_pts"], g["pib_boxes"]), g["pib_all"])
    assert (g["pib_all"].sum(2) > 1).any()                               # a point in two boxes: `first` keeps the lower index


def test_host_side_argument_checks():
    from sst_b200 import _lib as L, ops
    rois, pts, feats = torch.zeros((2, 7)), torch.zeros((5, 3)), torch.zeros((5, 4))
    with pytest.raises(L.SSTB200Error, match="out_size"):
        ops.RoIAwarePool3d(256)(rois, pts, feats)
    with pytest.raises(L.SSTB200Error, match="out_size"):
        ops.RoIAwarePool3d((14, 0, 14))(rois, pts, feats)
    with pytest.raises(L.SSTB200Error, match="max_pts_per_voxel"):
        ops.RoIAwarePool3d(14, max_pts_per_voxel=0)(rois, pts, feats)
    with pytest.raises(AssertionError):
        ops.RoIAwarePool3d(14, mode="sum")
    with pytest.raises(L.SSTB200Error, match="mode"):
        ops.RoIAwarePool3dFunction.apply(rois, pts, feats, 14, 128, 2)
    with pytest.raises(L.SSTB200Error, match="CUDA"):                   # CPU tensors raise: there is no CPU path
        ops.RoIAwarePool3d(14)(rois, pts, feats)
    with pytest.raises(L.SSTB200Error, match="CUDA"):
        ops.points_in_boxes_gpu(pts[None], rois[None])
    with pytest.raises(L.SSTB200Error, match="CUDA"):
        ops.points_in_boxes_batch(pts[None], rois[None])
    with pytest.raises(AssertionError):
        ops.points_in_boxes_gpu(pts[None], rois[None, :, :5])
