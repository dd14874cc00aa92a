"""GPU: FSD RoI point pooling (SURVEY 8f next-3) - sstb200_dynamic_point_pool through ops.dynamic_point_pool(_mixed) and
DynamicPointROIExtractor.  Point and RoI indices and the row count are BIT-EXACT against the oracle (oracle/roi_pool_oracle.dynamic_point_pool,
pinned to the reference's box test by tests/test_oracle_roi_pool_vs_reference.py), is_in_margin exact, local xyz / offsets within 1e-5 m;
membership also against the reference's own CUDA points_in_boxes_batch when oracle/_ref holds it."""
import math
import warnings

import pytest
import torch

from oracle import build_ref, roi_pool_oracle as RO, sst_oracle as O

pytestmark = pytest.mark.gpu
EXTRA = [0.5, 0.5, 0.5]


def _check(got, ref):
    idx, roi, feats = (t.cpu() for t in got)
    assert idx.dtype == torch.int64 and roi.dtype == torch.int64 and feats.dtype == torch.float32 and feats.shape[1] == 13
    assert idx.shape == ref[0].shape, (idx.shape, ref[0].shape)
    assert torch.equal(idx, ref[0]) and torch.equal(roi, ref[1])
    assert torch.equal(feats[:, :3], ref[2][:, :3]) and torch.equal(feats[:, 12], ref[2][:, 12])
    assert (feats[:, 3:12] - ref[2][:, 3:12]).abs().max().item() <= 1e-5


def _pool(rois, pts, *a, **k):
    from sst_b200 import ops
    return ops.dynamic_point_pool(rois.cuda(), pts.cuda(), *a, **k)


@pytest.fixture(scope="module")
def fsd_frame():
    pts, rois, _, _ = RO.synth_roi_frame(11, n_pts=100000, n_rois=500)
    return pts, rois, RO.dynamic_point_pool(rois, pts, EXTRA, 256)


def test_fsd_shape_vs_oracle_and_deterministic(cuda, fsd_frame):
    pts, rois, ref = fsd_frame
    a = _pool(rois, pts, EXTRA, 256)
    _check(a, ref)
    assert ref[0].numel() > 20000 and (ref[2][:, 12] == 1).any() and (ref[2][:, 12] == 0).any()
    b = _pool(rois, pts, EXTRA, 256)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_cap_keeps_lowest_indices_and_empty_rois(cuda):
    pts, rois, _, _ = RO.synth_roi_frame(12, n_pts=30000, n_rois=60, spread=20.0)
    big = torch.tensor([[0.0, 0.0, -3.0, 12.0, 12.0, 6.0, 0.3]])               # holds thousands of points
    far = rois[:5].clone()
    far[:, 0] += 500.0                                                         # no point inside
    rois = torch.cat([far[:2], big, rois, far[2:]])
    ref = RO.dynamic_point_pool(rois, pts, EXTRA, 64, max_all_pts=10**6)
    assert (ref[1] == 2).sum() == 64
    _check(_pool(rois, pts, EXTRA, 64, 10**6), ref)
    _check(_pool(rois, pts, [0.0, 0.0, 0.0], 3000, 10**6), RO.dynamic_point_pool(rois, pts, [0.0, 0.0, 0.0], 3000, max_all_pts=10**6))


def test_no_pair_gives_fake_row_and_capacity_cut(cuda):
    pts, rois, _, _ = RO.synth_roi_frame(13, n_pts=20000, n_rois=80, spread=15.0)
    far = rois.clone()
    far[:, 1] -= 800.0
    idx, roi, feats = _pool(far, pts, EXTRA, 32)
    assert idx.tolist() == [-1] and roi.tolist() == [-1] and int(feats.abs().sum()) == 0
    ref = RO.dynamic_point_pool(rois, pts, EXTRA, 32, max_all_pts=500)
    with pytest.warns(UserWarning, match="max_all_pts"):
        got = _pool(rois, pts, EXTRA, 32, 500)
    assert got[0].numel() == 500
    _check(got, ref)


def test_membership_vs_reference_cuda_kernel(cuda, fsd_frame):
    ref_mod = build_ref.load_module("roiaware_pool3d_ext_ref")
    if ref_mod is None:
        pytest.skip("oracle/_ref roiaware_pool3d build not present")
    pts, rois, _ = fsd_frame
    idx, roi, feats = (t.cpu() for t in _pool(rois, pts, EXTRA, 8192, 10**7))
    for boxes in (RO.enlarge_boxes(rois, EXTRA), rois):
        out = torch.zeros((1, pts.shape[0], rois.shape[0]), dtype=torch.int32, device=cuda)
        ref_mod.points_in_boxes_batch(boxes[None].contiguous().to(cuda), pts[None].contiguous().to(cuda), out)
        pairs = out[0].t().nonzero().cpu()                                   # (roi, point), roi-major, points ascending
        if boxes is rois:
            inner = feats[:, 12] == 0
            assert torch.equal(torch.stack([roi[inner], idx[inner]], 1), pairs)
        else:
            assert torch.equal(torch.stack([roi, idx], 1), pairs)


def test_mixed_op_equals_per_sample_calls(cuda):
    from sst_b200 import ops
    pts, rois, pb, rb = RO.synth_roi_frame(14, n_pts=60000, n_rois=240, spread=25.0, batch_size=3)
    got = [t.cpu() for t in ops.dynamic_point_pool_mixed(rois.cuda(), rb.cuda(), pts.cuda(), pb.cuda(), EXTRA, 128)]
    assert torch.equal(rb[got[1]], pb[got[0]])                              # no cross-sample pair
    parts, pbase, rbase = [], 0, 0
    for b in range(3):
        pm, rm = pb == b, rb == b
        i, r, f = (t.cpu() for t in ops.dynamic_point_pool(rois[rm].cuda(), pts[pm].cuda(), EXTRA, 128))
        if i[0] >= 0:
            parts.append((i + pbase, r + rbase, f))
        pbase, rbase = pbase + int(pm.sum()), rbase + int(rm.sum())
    for k in range(3):
        assert torch.equal(got[k], torch.cat([p[k] for p in parts]))
    _check(got, RO.dynamic_point_pool(rois, pts, EXTRA, 128, max_all_pts=200000, rois_batch=rb, pts_batch=pb))


def _reference_loop(ext, pts_xyz, batch_inds, rois, max_inbox_point):
    """dynamic_point_roi_extractor.py:53-109 composed from the single op"""
    from sst_b200 import ops
    all_inds, all_info, all_roi = [], [], []
    rbase = pbase = 0
    for b in range(int(batch_inds.max()) + 1):
        rm, pm = rois[..., 0].int() == b, batch_inds.int() == b
        nr, npt = int(rm.sum()), int(pm.sum())
        i, r, f = ops.dynamic_point_pool(rois[..., 1:][rm], pts_xyz[pm], ext.extra_wlh, max_inbox_point, ext.max_all_pts)
        if len(i) == 1 and i[0].item() == -1:
            all_inds.append(i), all_info.append(f), all_roi.append(r)
        else:
            all_inds.append(i + pbase), all_info.append(f), all_roi.append(r + rbase)
        pbase += npt
        rbase += nr
    info = torch.cat(all_info)
    return torch.cat(all_inds), torch.cat(all_roi), dict(local_xyz=info[:, 3:6], boundary_offset=info[:, 6:-1], is_in_margin=info[:, -1])


def _same(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k in ("local_xyz", "boundary_offset", "is_in_margin"):
        assert torch.equal(a[2][k], b[2][k]), k


def test_extractor_vs_reference_loop(cuda):
    import sst_b200
    from sst_b200 import _lib as L
    pts, rois, pb, rb = RO.synth_roi_frame(15, n_pts=40000, n_rois=150, spread=20.0, batch_size=3)
    rois7 = torch.cat([rb[:, None].float(), rois], 1)
    rois7[rb == 1, 2] += 900.0                                                 # sample 1: RoIs but no pair -> its own fake row
    p, b, r = pts.cuda(), pb.cuda(), rois7.cuda()
    ext = sst_b200.ROI_EXTRACTORS.build(dict(type="DynamicPointROIExtractor", extra_wlh=EXTRA, max_inbox_point=256, debug=False))
    got = ext(p, b, r)
    assert (got[0] == -1).sum() == 1
    _same(got, _reference_loop(ext, p, b, r, 256))
    # debug=True runs the reference's asserts (:92-101): they hold on real rows, and a fake row fails them there as here
    dbg = sst_b200.DynamicPointROIExtractor(extra_wlh=EXTRA, max_inbox_point=256, debug=True)
    r_all = torch.cat([rb[:, None].float(), rois], 1).cuda()
    _same(dbg(p, b, r_all), _reference_loop(dbg, p, b, r_all, 256))
    with pytest.raises(AssertionError):
        dbg(p, b, r)
    # per-sample capacity
    small = sst_b200.DynamicPointROIExtractor(extra_wlh=EXTRA, max_inbox_point=64, max_all_pts=700, debug=False)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        got, exp = small(p, b, r), _reference_loop(small, p, b, r, 64)
    assert (got[1] >= 0).sum() == 1400
    _same(got, exp)
    # batch_size == 1: one call, no bases
    one = ext(p[b == 0], torch.zeros_like(b[b == 0]), r[rb.cuda() == 0], batch_size=1)
    i, ri, f = sst_b200.ops.dynamic_point_pool(r[rb.cuda() == 0][:, 1:].contiguous(), p[b == 0], EXTRA, 256)
    assert torch.equal(one[0], i) and torch.equal(one[1], ri) and torch.equal(one[2]["boundary_offset"], f[:, 6:12])
    # errors
    with pytest.raises(L.SSTB200Error):
        ext(pts, pb, rois7)
    with pytest.raises(ValueError):
        ext(p, b, r.flip(0))
    no_roi = r[rb.cuda() != 2]
    with pytest.raises(ValueError):
        ext(p, b, no_roi)


def test_bbox_head_first_block_on_pooled_points(cuda):
    """FullySparseBboxHead's f_cluster (fsd_bbox_head.py:129-149: local_xyz, boundary offsets, is_in_margin, rel_xyz = 13 channels) from
    the extractor, through the fused fp32 SIRLayer of the head's first block (in 213, [128, 128], rel [16, 32])"""
    import sst_b200
    from sst_b200.sir_modules import SIRLayer
    pts, rois, pb, rb = RO.synth_roi_frame(16, n_pts=20000, n_rois=80, spread=15.0, batch_size=2)
    rois7 = torch.cat([rb[:, None].float(), rois], 1).cuda()
    ext = sst_b200.DynamicPointROIExtractor(extra_wlh=EXTRA, max_inbox_point=256, debug=True)
    inds, roi_inds, info = ext(pts.cuda(), pb.cuda(), rois7)
    assert (inds >= 0).all()
    xyz = pts.cuda()[inds]
    rel_xyz = xyz - rois7[roi_inds, 1:4]
    f_cluster = torch.cat([info["local_xyz"], info["boundary_offset"], info["is_in_margin"][:, None], rel_xyz], -1)
    assert f_cluster.shape[1] == 13
    torch.manual_seed(0)
    m = SIRLayer(in_channels=213, feat_channels=[128, 128], rel_mlp_hidden_dims=[16, 32], rel_mlp_in_channel=13,
                 norm_cfg=dict(type='LN', eps=1e-3), mode='max', return_point_feats=True, rel_dist_scaler=10.0,
                 xyz_normalizer=[20, 20, 4], act='gelu').eval()
    feats = torch.randn((xyz.shape[0], 210), generator=torch.Generator().manual_seed(3))
    x = torch.cat([xyz.cpu(), feats], 1)
    new_coors, inv = torch.unique(roi_inds.cpu(), return_inverse=True)
    w = {("x." + k): v for k, v in m.state_dict().items()}
    pf, gf = O.sir_layer_forward(x, inv, new_coors.shape[0], f_cluster.cpu(), w, "x.", 3, 2, [20, 20, 4], 1e-3, "gelu", 10.0)
    m = m.to(cuda)
    with torch.no_grad():
        a, b = m(x.to(cuda), roi_inds[:, None], f_cluster)
    for got, exp in ((a, pf), (b, gf)):
        err = (got.cpu() - exp).abs().max().item() / exp.abs().max().item()
        assert err < 1e-3, err


def test_cpu_tensors_raise():
    from sst_b200 import _lib as L, ops
    with pytest.raises(L.SSTB200Error):
        ops.dynamic_point_pool(torch.zeros((1, 7)), torch.zeros((4, 3)), EXTRA, 8)
