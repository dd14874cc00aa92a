"""GPU: points_in_boxes_gpu / points_in_boxes_batch and RoIAwarePool3d (sstb200_points_in_boxes, sstb200_roiaware_pool3d_*) through
ops and Single3DRoIAwareExtractor.  Membership and the forward are BITWISE equal to the reference's own CUDA kernels (oracle/_ref,
built by oracle/build_ref_roiaware.py) and to the oracle (oracle/roiaware_oracle.py); the compact saved state, expanded to the reference's
dense layout, equals the reference's; the backward is within 1e-6 of the reference's float atomics and bit-identical from run to run."""
import pytest
import torch

from oracle import build_ref, roi_pool_oracle as RO, roiaware_oracle as RA

pytestmark = pytest.mark.gpu
REF = build_ref.load_module("roiaware_pool3d_ext_ref")


def _bits(t):
    """fp32 as its bit patterns (so -0.0 != 0.0), every NaN as one pattern: NaN payloads differ between CPU and GPU arithmetic"""
    t = t.cpu().contiguous()
    if t.dtype != torch.float32:
        return t
    return torch.where(torch.isnan(t), torch.full_like(t, float("nan")), t).view(torch.int32)


def _ref_pib(points, boxes, first):
    points, boxes = points.cuda().contiguous(), boxes.cuda().contiguous()
    if first:
        out = torch.full(points.shape[:2], -1, dtype=torch.int32, device="cuda")
        REF.points_in_boxes_gpu(boxes, points, out)
    else:
        out = torch.zeros((*points.shape[:2], boxes.shape[1]), dtype=torch.int32, device="cuda")
        REF.points_in_boxes_batch(boxes, points, out)
    return out.cpu()


def _check_pib(points, boxes, with_ref=True):
    from sst_b200 import ops
    first = ops.points_in_boxes_gpu(points.cuda(), boxes.cuda()).cpu()
    every = ops.points_in_boxes_batch(points.cuda(), boxes.cuda()).cpu()
    assert first.dtype == torch.int32 and every.dtype == torch.int32
    assert first.shape == points.shape[:2] and every.shape == (*points.shape[:2], boxes.shape[1])
    assert torch.equal(first, RA.points_in_boxes_gpu(points, boxes))
    assert torch.equal(every, RA.points_in_boxes_batch(points, boxes))
    if with_ref and REF is not None:
        assert torch.equal(first, _ref_pib(points, boxes, True))
        assert torch.equal(every, _ref_pib(points, boxes, False))
    return first, every


def test_points_in_boxes_waymo_frame(cuda):
    pts, rois, _, _ = RO.synth_roi_frame(41, n_pts=150000, n_rois=200, spread=40.0)
    rois[::3, 3:6] *= 2.5                                                  # enlarged boxes overlap their neighbours
    first, every = _check_pib(pts[None], rois[None])
    assert (every.sum(2) > 1).sum() > 100 and (first >= 0).sum() > 30000


def test_points_in_boxes_batch_with_padding_boxes_and_faces(cuda):
    x = RA.golden_inputs()
    first, every = _check_pib(x["pib_pts"], x["pib_boxes"])
    assert every[1, :, 4:].sum() == 0                                     # zero-size padding boxes hold nothing
    pts, rois, _, _ = RO.synth_roi_frame(42, n_pts=30000, n_rois=100, spread=15.0)
    pts2, rois2, _, _ = RO.synth_roi_frame(43, n_pts=30000, n_rois=100, spread=15.0)
    rois2[60:] = 0.0
    _check_pib(torch.stack([pts, pts2]), torch.stack([rois, rois2]))
    _check_pib(x["pts"][None], x["rois"][None])                           # points on faces, overlapping boxes, an empty box


def test_points_in_boxes_empty(cuda):
    for B, M, T in ((2, 100, 0), (2, 0, 5), (0, 10, 3), (1, 0, 0)):
        pts, boxes = torch.randn((B, M, 3)), torch.rand((B, T, 7)) + 0.5
        first, every = _check_pib(pts, boxes, with_ref=False)              # the reference's launcher exits on a zero-block grid
        assert (first == -1).all() and every.numel() == B * M * T


def _ref_forward(rois, pts, feats, out_size, m, mode):
    ox, oy, oz = RA.out_size3(out_size)
    n, C = rois.shape[0], feats.shape[1]
    pooled = torch.zeros((n, ox, oy, oz, C), device="cuda")
    argmax = torch.zeros((n, ox, oy, oz, C), dtype=torch.int32, device="cuda")
    pidx = torch.zeros((n, ox, oy, oz, m), dtype=torch.int32, device="cuda")
    REF.forward(rois.cuda().contiguous(), pts.cuda().contiguous(), feats.cuda().contiguous(), argmax, pidx, pooled, mode)
    return pooled, argmax, pidx


def _ref_backward(pidx, argmax, grad_out, num_pts, mode):
    grad_in = torch.zeros((num_pts, grad_out.shape[-1]), device="cuda")
    REF.backward(pidx, argmax, grad_out.cuda().contiguous(), grad_in, mode)
    return grad_in


def _ours(rois, pts, feats, out_size, m, mode):
    from sst_b200 import ops
    return ops.roiaware_pool3d_forward(rois.cuda(), pts.cuda(), feats.cuda(), out_size, m, mode)


def _check_pool(rois, pts, feats, out_size, m, mode, grad=True):
    """forward bitwise against the reference and the oracle, state expanded to the reference's layout, backward"""
    from sst_b200 import ops
    pooled, state = _ours(rois, pts, feats, out_size, m, mode)
    o_pooled, o_arg, o_pidx = RA.roiaware_pool3d(rois, pts, feats, out_size, m, mode)
    assert torch.equal(_bits(pooled), _bits(o_pooled))
    slot, voff, pidx, argmax, counts, P = state
    dense_idx, dense_arg = RA.expand_state(slot.cpu(), voff.cpu(), pidx.cpu(), None if argmax is None else argmax.cpu(), counts.cpu(),
                                           rois.shape[0], out_size, m, feats.shape[1])
    assert torch.equal(dense_idx, o_pidx)
    if mode == 0:
        assert torch.equal(dense_arg, o_arg)
    g = torch.randn(pooled.shape, generator=torch.Generator().manual_seed(7))
    gin = ops.roiaware_pool3d_backward(g.cuda(), state, pts.shape[0], mode) if grad else None
    if grad:
        assert torch.equal(_bits(gin), _bits(ops.roiaware_pool3d_backward(g.cuda(), state, pts.shape[0], mode)))   # run to run
        o_gin = RA.roiaware_pool3d_backward(o_pidx, o_arg, g, pts.shape[0], mode)
        torch.testing.assert_close(gin.cpu(), o_gin, rtol=1e-6, atol=1e-7 * max(1.0, o_gin.abs().max().item()))
    if REF is not None:
        r_pooled, r_arg, r_pidx = _ref_forward(rois, pts, feats, out_size, m, mode)
        assert torch.equal(_bits(pooled), _bits(r_pooled))
        assert torch.equal(dense_idx, r_pidx.cpu())
        if mode == 0:
            assert torch.equal(dense_arg, r_arg.cpu())
        if grad:
            r_gin = _ref_backward(r_pidx, r_arg, g, pts.shape[0], mode).cpu()
            torch.testing.assert_close(gin.cpu(), r_gin, rtol=1e-6, atol=1e-7 * max(1.0, r_gin.abs().max().item()))
    return pooled, state


def _parta2_frame(seed, n_pts=16000, n_rois=64, spread=15.0):
    pts, rois, _, _ = RO.synth_roi_frame(seed, n_pts=n_pts, n_rois=n_rois, spread=spread)
    return pts, rois


@pytest.mark.parametrize("mode", [0, 1])
def test_pool3d_parta2_shape(cuda, mode):
    pts, rois = _parta2_frame(51)
    feats = torch.randn((pts.shape[0], 16 if mode == 0 else 4), generator=torch.Generator().manual_seed(1))
    pooled, state = _check_pool(rois, pts, feats, 14, 128, mode)
    assert int(state[4][0]) > 1000 and pooled.abs().sum() > 0


@pytest.mark.parametrize("mode", [0, 1])
def test_pool3d_edge_cases(cuda, mode):
    x = RA.golden_inputs()
    rois, pts, feats = x["rois"], x["pts"], x["feats"]                   # overlaps, faces, a crowded voxel, ties, NaN, -inf
    for out_size, m in (((6, 4, 3), 8), (14, 1), (14, 1000), (1, 128), ((1, 1, 1), 3), ((255, 1, 1), 16), ((2, 255, 3), 4)):
        _check_pool(rois, pts, feats, out_size, m, mode)
    allneg = torch.full_like(feats, -float("inf"))
    allneg[::2] = float("nan")
    pooled, state = _check_pool(rois, pts, allneg, (6, 4, 3), 8, mode)
    if mode == 0:
        assert (pooled == 0).all() and (state[3][:int(state[4][0])] == -1).all()


def test_pool3d_empty_inputs(cuda):
    from sst_b200 import ops
    x = RA.golden_inputs()
    for rois, pts in ((x["rois"][:0], x["pts"]), (x["rois"], x["pts"][:0]), (x["rois"][5:], x["pts"])):
        feats = torch.randn((pts.shape[0], 3))
        pooled, state = ops.roiaware_pool3d_forward(rois.cuda(), pts.cuda(), feats.cuda(), (4, 3, 2), 8, 0)
        assert pooled.shape == (rois.shape[0], 4, 3, 2, 3) and (pooled == 0).all() and state[5] == 0
        gin = ops.roiaware_pool3d_backward(torch.ones_like(pooled), state, pts.shape[0], 0)
        assert gin.shape == (pts.shape[0], 3) and (gin == 0).all()


def test_pool3d_autograd_and_module(cuda):
    from sst_b200 import ops
    pts, rois = _parta2_frame(52, n_pts=8000, n_rois=32)
    feats = torch.randn((pts.shape[0], 16), generator=torch.Generator().manual_seed(2)).cuda().requires_grad_()
    for mode in ("max", "avg"):
        layer = ops.RoIAwarePool3d((10, 8, 6), max_pts_per_voxel=32, mode=mode)
        out = layer(rois.cuda(), pts.cuda(), feats)
        g = torch.randn(out.shape, device="cuda")
        (grad,) = torch.autograd.grad(out, feats, g)
        pooled, state = ops.roiaware_pool3d_forward(rois.cuda(), pts.cuda(), feats.detach(), (10, 8, 6), 32, layer.mode)
        assert torch.equal(_bits(out.detach()), _bits(pooled))
        assert torch.equal(_bits(grad), _bits(ops.roiaware_pool3d_backward(g, state, pts.shape[0], layer.mode)))


def test_library_argument_errors(cuda):
    import ctypes as C
    from sst_b200 import _lib as L
    pts = torch.zeros((4, 3), device="cuda")
    rois = torch.ones((2, 7), device="cuda")
    nb = torch.tensor([0, -1], dtype=torch.int32, device="cuda")
    c = L.ctx(pts.device)
    P = C.c_int64()

    def plan(out=(4, 4, 4), m=8, rb=None, pb=None, R=2, N=4):
        return L.lib().sstb200_roiaware_pool3d_plan(c, rois.data_ptr(), L.ptr(rb), R, pts.data_ptr(), L.ptr(pb), N, L.arr(C.c_int32, list(out)),
                                                    m, C.byref(P))
    assert plan((256, 4, 4)) == -2 and plan((4, 0, 4)) == -2 and plan(m=0) == -2 and plan(R=-1) == -2
    assert plan(rb=nb, pb=torch.zeros(4, dtype=torch.int32, device="cuda")) == -2
    assert plan(rb=torch.zeros(2, dtype=torch.int32, device="cuda"), pb=torch.tensor([0, 0, -3, 0], dtype=torch.int32, device="cuda")) == -2
    assert plan(out=(255, 255, 255), R=1 << 21, N=1 << 20) == -3            # 21 + 24 + 20 > 64 key bits: refused before any work
    assert plan() == 0
    out = torch.empty(8, device="cuda")
    assert L.lib().sstb200_roiaware_pool3d_forward(c, pts.data_ptr(), 1, 5, out.data_ptr(), out.data_ptr(), out.data_ptr(), out.data_ptr(),
                                                   out.data_ptr(), out.data_ptr()) == -2   # bad mode
    assert L.lib().sstb200_roiaware_pool3d_forward(c, pts.data_ptr(), 1, 0, out.data_ptr(), out.data_ptr(), out.data_ptr(), out.data_ptr(),
                                                   out.data_ptr(), out.data_ptr()) == -2   # no plan directly before it
    assert L.lib().sstb200_points_in_boxes(c, pts.data_ptr(), rois.data_ptr(), 1, 4, 2, 3, out.data_ptr()) == -2


def _reference_extractor(feats, coordinate, batch_inds, rois, out_size, m, mode):
    """single_roiaware_extractor.py:31-53 over the reference's own forward"""
    out = []
    for b in range(int(batch_inds.max()) + 1):
        ri, ci = rois[..., 0].int() == b, batch_inds.int() == b
        out.append(_ref_forward(rois[..., 1:][ri], coordinate[ci], feats[ci], out_size, m, mode)[0])
    return torch.cat(out, 0)


@pytest.mark.parametrize("mode", ["max", "avg"])
def test_extractor_vs_reference_loop(cuda, mode):
    import sst_b200
    pts, rois, pb, rb = RO.synth_roi_frame(53, n_pts=24000, n_rois=96, spread=15.0, batch_size=3)
    perm = torch.randperm(rois.shape[0], generator=torch.Generator().manual_seed(4))
    rois8 = torch.cat([rb[:, None].float(), rois], 1)[perm]                  # RoI batch ids unsorted
    rois8 = torch.cat([rois8, rois8[:3] * torch.tensor([0.0] + [1.0] * 7) + torch.tensor([7.0] + [0.0] * 7)])   # batch 7: no points
    feats = torch.randn((pts.shape[0], 16), generator=torch.Generator().manual_seed(5))
    ext = sst_b200.ROI_EXTRACTORS.build(dict(type="Single3DRoIAwareExtractor",
                                             roi_layer=dict(type="RoIAwarePool3d", out_size=(8, 6, 4), max_pts_per_voxel=32, mode=mode)))
    got = ext(feats.cuda(), pts.cuda(), pb.cuda(), rois8.cuda())
    exp = RA.single_roiaware_extractor(feats, pts, pb, rois8, (8, 6, 4), 32, ext.roi_layer.mode)
    assert got.shape == exp.shape == (96, 8, 6, 4, 16)
    assert torch.equal(_bits(got), _bits(exp))
    if REF is not None:
        assert torch.equal(_bits(got), _bits(_reference_extractor(feats.cuda(), pts.cuda(), pb.cuda(), rois8.cuda(), (8, 6, 4), 32,
                                                                  ext.roi_layer.mode)))
    f = feats.cuda().requires_grad_()
    out = ext(f, pts.cuda(), pb.cuda(), rois8.cuda())
    (g,) = torch.autograd.grad(out, f, torch.ones_like(out))
    assert g.abs().sum() > 0
