"""GPU: rotated BEV overlap / IoU / NMS (sstb200_boxes_{overlap,iou}_bev, sstb200_nms_bev) through ops.boxes_iou_bev, boxes_overlap_bev,
nms_gpu, nms_normal_gpu and box3d_multiclass_nms.  IoU and overlap against the float64 oracle (oracle/iou3d_oracle.py, pinned to the
reference by tests/test_oracle_iou3d_vs_reference.py) and, when oracle/_ref holds it, the reference's own CUDA build; keep lists
identical to both on box sets with no IoU within 1e-4 of the threshold."""
import ctypes as C
import json
import types

import numpy as np
import pytest
import torch

from oracle import build_ref, iou3d_oracle as IO

pytestmark = pytest.mark.gpu
REF = build_ref.load_module("iou3d_ref")
THRESHOLDS = (0.01, 0.25, 0.7)
# The reference (fp32, absolute coordinates, angle-sorted polygon) against the fp64 oracle, measured on an H100: the dense, spread and
# special sets stay within 1.4e-5, but for sub-metre boxes 75 m from the origin 70 of 748 overlapping pairs exceed 5e-5 (worst |dIoU|
# 0.667), and for zero-area boxes it returns garbage (IoU 3.09 and 30.85 seen).  So the fp64 oracle is the binding check; zero-area boxes
# are left out of the reference comparison, at most a quarter of the overlapping pairs may exceed 5e-5, and none the observed maximum.
REF_TOL, REF_TOL_MAX, REF_FRAC = 5e-5, 0.67, 0.25
OBSERVED = {}


def _ops():
    from sst_b200 import ops
    return ops


def _record(key, value):
    """worst observed deviations, printed when the module finishes (visible with `pytest -s`)"""
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), float(value))


@pytest.fixture(scope="module", autouse=True)
def _report_observed():
    yield
    if OBSERVED:
        print("\n[iou3d observed] " + json.dumps(OBSERVED, indent=1, sort_keys=True))


def ref_matrix(fn, a, b):
    out = torch.zeros((a.shape[0], b.shape[0]), device="cuda")
    getattr(REF, fn)(a.cuda().contiguous(), b.cuda().contiguous(), out)
    return out.cpu()


def ref_nms(boxes, scores, thresh, rotated=True, pre_maxsize=None, post_max_size=None):
    """iou3d_utils.py:31-56 / 106-124 over the reference extension"""
    boxes, scores = boxes.cuda(), scores.cuda()
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    b = boxes[order].contiguous()
    keep = torch.zeros(b.size(0), dtype=torch.long)
    num = (REF.nms_gpu if rotated else REF.nms_normal_gpu)(b, keep, float(thresh), b.device.index)
    keep = order[keep[:num].cuda()].contiguous()
    if post_max_size is not None:
        keep = keep[:post_max_size]
    return keep.cpu()


def _check_matrices(a, b, label):
    ops = _ops()
    iou, ov = ops.boxes_iou_bev(a.cuda(), b.cuda()).cpu(), ops.boxes_overlap_bev(a.cuda(), b.cuda()).cpu()
    assert iou.dtype == torch.float32 and iou.shape == (a.shape[0], b.shape[0]) and ov.shape == iou.shape
    assert torch.isfinite(iou).all() and torch.isfinite(ov).all()
    oi, oo = IO.boxes_iou_bev(a, b), IO.boxes_overlap_bev(a, b)
    d_iou = (iou.double() - oi).abs().max().item()
    d_ov = ((ov.double() - oo).abs() - 1e-5 * oo.abs()).max().item()
    _record("iou_vs_fp64", d_iou)
    _record("overlap_vs_fp64_minus_rel", d_ov)
    assert d_iou <= 1e-5, d_iou
    assert d_ov <= 1e-5, d_ov
    if REF is not None:
        r_iou, r_ov = ref_matrix("boxes_iou_bev_gpu", a, b).double(), ref_matrix("boxes_overlap_bev_gpu", a, b).double()
        area = lambda x: ((x[:, 2] - x[:, 0]) * (x[:, 3] - x[:, 1])) != 0
        ok = area(a)[:, None] & area(b)[None, :]
        d = (r_iou - oi).abs()[ok]
        _record(f"reference_iou_vs_fp64_{label}", d.max().item())
        _record("reference_overlap_vs_fp64", ((r_ov - oo).abs() / oo.abs().clamp(min=1.0))[ok].max().item())
        _record(f"reference_pairs_over_5e-5_{label}", (d > REF_TOL).sum().item())
        _record(f"reference_overlapping_pairs_{label}", (oi[ok] > 0).sum().item())
        assert d.max().item() <= REF_TOL_MAX and (d > REF_TOL).sum().item() <= REF_FRAC * max(1, (oi[ok] > 0).sum().item())
    return iou, ov


def test_iou_and_overlap_vs_oracle_and_reference(cuda):
    dense = IO.synth_boxes(1, 1200, objects=80)                        # overlapping proposals, centres within +-75 m
    _check_matrices(dense[:600], dense[600:], "dense")
    _check_matrices(IO.synth_boxes(2, 700), IO.synth_boxes(3, 500), "spread")    # spread: mostly the exact-zero early-out
    tiny = IO.synth_boxes(4, 400, objects=30)
    tiny[:, 2:4] = tiny[:, :2] + (tiny[:, 2:4] - tiny[:, :2]) * 0.05  # sub-metre boxes far from the origin
    _check_matrices(tiny, tiny, "tiny")


def test_special_cases(cuda):
    sp = IO.special_boxes()
    iou, ov = _check_matrices(sp, sp, "special")
    for i, j in ((0, 1), (19, 20)):                                     # identical, near the origin and 70 m from it
        assert abs(iou[i, j].item() - 1.0) <= 1e-6 and abs(iou[j, i].item() - 1.0) <= 1e-6
    assert abs(iou[0, 0].item() - 1.0) <= 1e-6
    zero = [16, 17, 18]                                                 # zero-area boxes: 0, never NaN
    assert (ov[zero] == 0).all() and (ov[:, zero] == 0).all() and (iou[zero] == 0).all() and (iou[:, zero] == 0).all()
    assert ov[3, 4].item() <= 1e-5                                      # touching along a shared edge
    assert abs(ov[0, 2].item() - 2.0) <= 1e-5                           # nested: the inner box's area


def test_empty_outputs(cuda):
    ops = _ops()
    a = IO.synth_boxes(5, 7).cuda()
    assert ops.boxes_iou_bev(a, a[:0]).shape == (7, 0) and ops.boxes_overlap_bev(a[:0], a).shape == (0, 7)


# ---- NMS ----------------------------------------------------------------------------------------------------------------------------
_SETS = {}


def nms_set(n, kind):
    """n boxes (+ distinct scores) with no pair whose fp64 IoU, rotated or axis-aligned, lies within 1e-4 of a tested threshold, and the
    fp64 pair values of the score-sorted list"""
    key = (n, kind)
    if key not in _SETS:
        m = int(n * (2.0 if kind == "sparse" else 1.3)) + 8     # spread boxes overlap often at 20k: more are dropped
        boxes = IO.synth_boxes(100 + n, m) if kind == "sparse" else IO.synth_boxes(200 + n, m, objects=max(1, m // 12))
        ok = np.intersect1d(IO.drop_near_threshold(boxes, THRESHOLDS).numpy(), IO.drop_near_threshold(boxes, THRESHOLDS, rotated=False).numpy())
        assert len(ok) >= n, (len(ok), n)
        boxes = boxes[torch.from_numpy(ok[:n])]
        scores = IO.distinct_scores(300 + n, n)
        order = scores.sort(0, descending=True)[1]
        pairs = {rot: IO.pair_values(boxes[order], boxes[order], "iou" if rot else "normal", upper=True) for rot in (True, False)}
        _SETS[key] = (boxes, scores, order, pairs)
    return _SETS[key]


def _reference_ious_near(boxes, thresh):
    """number of the reference's own fp32 rotated IoUs within 1e-4 of the threshold (the fp64 IoUs keep 1e-4 away by construction, so
    these are the reference's polygon failures; where there are none its keep list is well defined)"""
    b = boxes.cuda().contiguous()
    near = 0
    for s in range(0, b.shape[0], 2048):
        m = torch.zeros((min(2048, b.shape[0] - s), b.shape[0]), device="cuda")
        REF.boxes_iou_bev_gpu(b[s:s + 2048].contiguous(), b, m)
        m[torch.arange(m.shape[0]), torch.arange(s, s + m.shape[0])] = 10.0
        near += int(((m - thresh).abs() < 1e-4).sum().item())
    return near


@pytest.mark.parametrize("kind", ["sparse", "dense"])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 1000, 4097, 20000])
def test_nms_keep_lists(cuda, n, kind):
    ops = _ops()
    boxes, scores, order, pairs = nms_set(n, kind)
    for t in THRESHOLDS:
        for rot in (True, False):
            got = (ops.nms_gpu(boxes.cuda(), scores.cuda(), t) if rot else ops.nms_normal_gpu(boxes.cuda(), scores.cuda(), t)).cpu()
            assert got.dtype == torch.int64
            want = order[IO.greedy_scan(n, *pairs[rot], t)]
            assert torch.equal(got, want), (t, rot, got.numel(), want.numel())
            if REF is not None and n > 0:
                near = _reference_ious_near(boxes[order], t) if rot else 0
                _record(f"reference_ious_near_threshold_n{n}_{kind}_{t}", near)
                if near == 0:
                    assert torch.equal(got, ref_nms(boxes, scores, t, rot)), (t, rot)


def test_nms_pre_and_post_max_size(cuda):
    ops = _ops()
    boxes, scores, order, _ = nms_set(20000, "dense")
    for pre, post in ((4096, 500), (None, 100), (1000, None)):
        for t in THRESHOLDS:
            got = ops.nms_gpu(boxes.cuda(), scores.cuda(), t, pre_maxsize=pre, post_max_size=post).cpu()
            want = IO.nms_gpu(boxes, scores, t, pre_maxsize=pre, post_max_size=post)
            assert torch.equal(got, want), (pre, post, t)
            if REF is not None:
                assert torch.equal(got, ref_nms(boxes, scores, t, True, pre, post))


def test_iou_equal_to_threshold_does_not_suppress(cuda):
    ops = _ops()
    boxes = torch.tensor([[0, 0, 2, 1, 0.0], [1, 0, 3, 1, 0.0]])        # overlap 1, union 3: IoU = fl(1/3), the threshold below
    scores = torch.tensor([0.9, 0.8])
    t = float(np.float32(1.0 / 3.0))
    assert ops.boxes_iou_bev(boxes.cuda(), boxes.cuda())[0, 1].item() == t
    for fn in (ops.nms_gpu, ops.nms_normal_gpu):
        assert fn(boxes.cuda(), scores.cuda(), t).tolist() == [0, 1]
        assert fn(boxes.cuda(), scores.cuda(), t * 0.999).tolist() == [0]
    assert IO.nms_gpu(boxes, scores, t).tolist() == [0, 1]


def test_two_calls_bit_identical(cuda):
    ops = _ops()
    boxes, scores, _, _ = nms_set(4097, "dense")
    b, s = boxes.cuda(), scores.cuda()
    assert torch.equal(ops.nms_gpu(b, s, 0.25), ops.nms_gpu(b, s, 0.25))
    assert torch.equal(ops.boxes_iou_bev(b, b), ops.boxes_iou_bev(b, b))


def test_segmented_equals_per_segment(cuda):
    ops = _ops()
    sizes = [0, 1, 64, 65, 3000, 0, 700, 129]
    threshs = [0.3, 0.1, 0.5, None, 0.25, 0.7, 0.01, 0.6]
    g = torch.Generator().manual_seed(7)
    segs = []
    for k, n in enumerate(sizes):
        b = IO.synth_boxes(400 + k, n, objects=max(1, n // 10))
        segs.append(b[torch.rand(n, generator=g).sort(descending=True)[1]])
    boxes = torch.cat(segs).cuda()
    offsets = [0]
    for n in sizes:
        offsets.append(offsets[-1] + n)
    for rot in (True, False):
        got = ops.nms_bev(boxes, offsets, threshs, rotated=rot).cpu()
        want = torch.cat([ops.nms_bev(boxes[offsets[k]:offsets[k + 1]], [0, n], [threshs[k]], rotated=rot).cpu() + offsets[k]
                          for k, n in enumerate(sizes)])
        assert torch.equal(got, want)
        assert torch.equal(got[(got >= offsets[3]) & (got < offsets[4])], torch.arange(offsets[3], offsets[4]))   # nms_thr None


def _mlvl(seed, n, num_classes=3):
    g = torch.Generator().manual_seed(seed)
    boxes = IO.synth_boxes(seed, int(n * 1.3), objects=max(1, n // 10))
    keep = np.intersect1d(IO.drop_near_threshold(boxes, (0.1, 0.25, 0.5, 0.7)).numpy(),
                          IO.drop_near_threshold(boxes, (0.1, 0.25, 0.5, 0.7), rotated=False).numpy())[:n]
    bfn = boxes[torch.from_numpy(keep)]
    n = bfn.shape[0]
    bboxes = torch.cat([(bfn[:, :2] + bfn[:, 2:4]) / 2, torch.rand(n, 5, generator=g)], 1)   # 7-dof boxes, content irrelevant
    scores = (torch.randperm(n * (num_classes + 1), generator=g).double() / (n * (num_classes + 1))).float().view(n, num_classes + 1)
    dirs = torch.rand(n, generator=g)
    attrs = torch.randint(0, 9, (n,), generator=g)
    b2d = torch.rand(n, 4, generator=g)
    return bboxes, bfn, scores, dirs, attrs, b2d


def _cmp(got, want):
    assert len(got) == len(want)
    for x, y in zip(got, want):
        assert x.dtype == y.dtype and x.shape == y.shape, (x.dtype, y.dtype, x.shape, y.shape)
        assert torch.equal(x.cpu(), y.cpu())


@pytest.mark.parametrize("rotate", [True, False])
def test_box3d_multiclass_nms(cuda, rotate):
    ops = _ops()
    bboxes, bfn, scores, dirs, attrs, b2d = _mlvl(31, 2000)
    ref_nms_fns = {}
    if REF is not None:
        ref_nms_fns = dict(nms_gpu=lambda b, s, t: ref_nms(b, s, t, True).to(b.device),
                           nms_normal_gpu=lambda b, s, t: ref_nms(b, s, t, False).to(b.device))
    cases = [
        ([0.1, 0.3, 0.2], dict(nms_thr=[0.25, 0.1, 0.5]), 500, (dirs,)),
        (0.2, dict(nms_thr=0.25), 100000, (dirs, attrs, b2d)),
        ([0.1, 0.3, 0.2], dict(nms_thr=[0.25, None, 0.7]), 100000, ()),
        (0.5, dict(nms_thr=0.1), 50, (dirs,)),                         # the max_num cut
        (2.0, dict(nms_thr=0.25), 500, (dirs, attrs, b2d)),             # everything below the score threshold
    ]
    for score_thr, c, max_num, extra in cases:
        cfg = types.SimpleNamespace(use_rotate_nms=rotate, **c)
        kw = dict(zip(("mlvl_dir_scores", "mlvl_attr_scores", "mlvl_bboxes2d"), extra))
        got = ops.box3d_multiclass_nms(bboxes.cuda(), bfn.cuda(), scores.cuda(), score_thr, max_num, cfg,
                                       **{k: v.cuda() for k, v in kw.items()})
        assert all(t.is_cuda for t in got)
        _cmp(got, IO.box3d_multiclass_nms(bboxes, bfn, scores, score_thr, max_num, cfg, **kw))
        if REF is not None:
            _cmp(got, IO.box3d_multiclass_nms(bboxes.cuda(), bfn.cuda(), scores.cuda(), score_thr, max_num, cfg,
                                              **{k: v.cuda() for k, v in kw.items()}, **ref_nms_fns))


def test_cpu_tensors_raise():
    from sst_b200 import _lib, ops
    b, s = IO.synth_boxes(6, 10), torch.rand(10)
    for call in (lambda: ops.boxes_iou_bev(b, b), lambda: ops.boxes_overlap_bev(b, b), lambda: ops.nms_gpu(b, s, 0.1),
                 lambda: ops.nms_normal_gpu(b, s, 0.1),
                 lambda: ops.box3d_multiclass_nms(b, b, torch.rand(10, 4), 0.1, 10, types.SimpleNamespace(nms_thr=0.1, use_rotate_nms=True))):
        with pytest.raises(_lib.SSTB200Error):
            call()


def test_argument_errors(cuda):
    from sst_b200 import _lib, ops
    L, c = _lib.lib(), _lib.ctx(cuda)
    nbytes = C.c_int64()

    def query(num, offs):
        return L.sstb200_nms_bev_workspace_bytes(c, num, _lib.arr(C.c_int32, offs), len(offs) - 1, C.byref(nbytes))

    assert query(10, [0, 4, 10]) == 0 and nbytes.value > 0
    assert query(-1, [0, -1]) == -2                                    # negative size
    assert query(10, [0, 6, 4, 10]) == -2                              # offsets decrease
    assert query(10, [0, 4, 9]) == -2                                  # do not end at num
    assert query(70000, [0, 70000]) == -3                              # a segment over the 65536-box limit
    b = IO.synth_boxes(8, 10).cuda()
    keep, num = torch.empty(10, dtype=torch.int64, device=cuda), torch.empty(1, dtype=torch.int32, device=cuda)
    assert query(10, [0, 10]) == 0
    args = (c, b.data_ptr(), 10, _lib.arr(C.c_int32, [0, 10]), 1, _lib.arr(C.c_float, [0.1]), 1)
    assert L.sstb200_nms_bev(*args, None, nbytes.value, keep.data_ptr(), num.data_ptr(), None) == -2   # NULL workspace
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=cuda)
    assert L.sstb200_nms_bev(*args, ws.data_ptr(), nbytes.value - 1, keep.data_ptr(), num.data_ptr(), None) == -4
    assert L.sstb200_boxes_iou_bev(c, b.data_ptr(), -1, b.data_ptr(), 10, keep.data_ptr()) == -2
    with pytest.raises(_lib.SSTB200Error):
        ops.nms_bev(b, [0, 5, 3, 10], [0.1, 0.1, 0.1])
    with pytest.raises(_lib.SSTB200Error):
        ops.nms_gpu(torch.zeros(70000, 5, device=cuda), torch.rand(70000, device=cuda), 0.1)
