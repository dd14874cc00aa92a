"""GPU: CenterHead's training kernels (sst_b200/csrc/centerpoint.cu) against the float64 / CPU oracle (oracle/centerpoint_oracle.py) at
the map shapes, slot cuts, grid sizes and clamp edges where they could go wrong.

Routes and edges
  targets   cp_slots_kernel (one 256-thread CTA per (sample, task), a ballot scan over the sample's boxes, class by class, cut at max_objs),
            cp_zero_heatmaps_kernel (float4 when B * ncls * H * W % 4 == 0 and the heatmap is 16-byte aligned, else scalar),
            cp_draw_kernel (the clipped (2r + 1)^2 window, combined by an integer max):
              maps W x H = 200x136, 136x200, 3x200, 150x1, 2x3, 135x201 (odd H W with odd B ncls: the scalar zero path), 800x544 grid at
              out_size_factor 1, 2, 4 and 8; gaussian_overlap 0.1 and 0.7; min_radius 0 (radius-0 boxes draw one cell of 1.0), 2 and 40
              (above every computed radius); norm_bbox False; box_dim 7 and 9;
              per-class counts 0, 1, 31, 32, 33, 255, 256, 257 and 513 in one sample, classes interleaved in input order, cut by max_objs
              = 1, inside a warp, on a warp edge, on a 256-box chunk edge, on a class boundary, and not at all;
              1, 6 and 16 tasks with uneven class counts, labels below 0 and past the last task; B = 1, 33 and 256 with empty samples
              first, in the middle and last, and a batch with no boxes; 17 tasks and B = 257 raise;
              centres on every edge and corner of a non-square map with windows past the edge, (-1, 0) cells and the last cell; 200
              overlapping same-class windows (bit-identical twice); a box at the 2^30 radius cap, whose class map is exactly 1.0
              everywhere (checked in closed form: exp(-d^2 / 2 sigma^2) rounds to 1 for every d on the map);
              outputs pre-filled with NaN / 0xFF through the C ABI, one heatmap at a one-float offset: every element is rewritten.
            Contract: ind, mask and anno_box[0, 1, 2, 8, 9] bit-exact; anno_box[3:8] within 1e-6; heatmap support and 1.0 centres exact,
            every other value within 1 ulp.
  focal     fl_forward_kernel / fl_backward_kernel, a grid of ceil(n / 2048) 256-thread blocks capped at 8 SMs (S = the device's SM
            count): n = 1, 255, 256, 257, 2047, 2048, 2049, 16384 S - 1, 16384 S, 16384 S + 1 and 49152 S + 5 (the capped grid, more than
            8 elements per thread); targets of exactly 1, nextafter(1, 0), 0 and 1e-30, logits of +-inf and NaN; loss_weight 1.5, an
            upstream gradient of 2^16 and fp16 logits; the clamp bounds swept at logit(1e-4) one logit ulp at a time and at logit(0.9999)
            one sigmoid ulp at a time (+-64 ulps each).
            Contract: num_pos exact; the loss within LOSS_C times its elements' summed first-order error (as for the gradient) of the
            float64 oracle's (a fixed relative bound does not fit: near the clamp one element's fp32 loss is off by 1e-4 relative, in the
            reference's fp32 as well); every gradient element within FL_GRAD_C * e of the
            oracle's, e the first-order fp32 error of the kernel's arithmetic: the sigmoid's relative error 2^-21 pushed through the
            derivative, 2^-20 of each term's size, and the rounding of 1 - p (2^-25 absolute for p <= 1/2) pushed through log(1 - p),
            which near p = 1e-4 is about 2e-4 of the gradient and is in the reference's fp32 as well.  Outside FL_BAND sigmoid ulps of a
            bound the clamp follows the oracle (inclusive); inside, the gradient is 0 or the unclamped value, except where the kernel's
            fp32 sigmoid is fixed by its arithmetic (at the upper bound, 1 + exp(-x) away from an fp32 rounding tie), where it must follow
            the fp32 inclusive rule.  A NaN logit gives a NaN loss and a NaN gradient at that element only.
  L1        l1_forward_kernel (one block) / l1_backward_kernel (one CTA per sample; the first masked slot of a cell writes the cell's sum in
            slot order): max_objs = 1, 255, 256, 257 and 4096 (4097 raises) with B up to 17 on 53x37 and 37x53 maps, ind 0 and H W - 1,
            random collisions, one cell shared by slots 0, 255, 256 and 300 and twenty shared by slots 260 + i, 516 + i and 3000 + i; every
            mask 0; NaN targets; zero code weights; a NaN prediction at a masked-out slot's cell.
            Contract: the loss within L1_RTOL of the float64 oracle (NaN where the oracle's is); every gradient element within
            L1_GRAD_C * (k + 2) 2^-24 times the cell's sum of |d loss / d pred| over its k slots (two roundings of each term, one per
            addition), exactly 0 where no slot contributes.
  module    CenterHead.loss and get_bboxes on a non-square two-task geometry against the oracle.

Bounds, with the worst errors seen on an NVIDIA H100 80GB HBM3 at a 700 W power limit (the file runs in about 25 s there):
  targets          the contract above                                            held with 0 ulp
  LOSS_C 0.25      focal loss, in units of its elements' summed first-order error  0.070 (relative 1.3e-5 on the clamp sweep, 2.9e-6
                                                                                   at n = 255, 6.8e-7 at n = 49152 S + 5)
  FL_GRAD_C 2      focal gradient, in units of e                                 0.989 (the 1 - p rounding, near p = 1e-4)
  FL_BAND 4        sigmoid ulps of undecided clamp around each bound             (expf is within 2 ulp)
  L1_RTOL 2.5e-7   L1 loss, relative (2^-22: two fp32 roundings per term)        4.2e-8
  L1_GRAD_C 0.6    L1 gradient, in units of (k + 2) 2^-24 of the absolute sum    0.300"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import centerpoint_oracle as CO
from oracle import iou3d_oracle as IO

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")

LOSS_C = 0.25           # focal loss, in units of the summed first-order error of its elements
FL_GRAD_C = 2.0         # focal gradient, in units of the first-order error e
FL_BAND = 4             # sigmoid ulps around each clamp bound
L1_RTOL = 2.5e-7        # L1 loss, relative
L1_GRAD_C = 0.6         # L1 gradient, in units of (slots + 2) 2^-24 of the cell's absolute sum
LO, HI = 1e-4, 1 - 1e-4
ULP_LO, ULP_HI = 2.0 ** -37, 2.0 ** -24      # fp32 spacing at 1e-4 and at 0.9999


# ---------------------------------------------------------------------------------------------------------------------------------------
# targets
# ---------------------------------------------------------------------------------------------------------------------------------------
def _boxes(g, G, cells, size=(0.5, 4.0)):
    """gravity-centred fp32 boxes [n, box_dim] centred at map coordinates cells [n, 2] (float64), sizes uniform in metres"""
    cfg = G['train_cfg']
    pc, vs, osf = cfg['point_cloud_range'], cfg['voxel_size'], cfg['out_size_factor']
    n = cells.shape[0]
    rows = [(pc[0] + cells[:, 0] * (vs[0] * osf))[:, None], (pc[1] + cells[:, 1] * (vs[1] * osf))[:, None],
            torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1,
            size[0] + torch.rand(n, 3, generator=g, dtype=torch.float64) * (size[1] - size[0]),
            (torch.rand(n, 1, generator=g, dtype=torch.float64) * 2 - 1) * math.pi]
    if G['box_dim'] == 9:
        rows.append(torch.randn(n, 2, generator=g, dtype=torch.float64) * 3)
    return torch.cat(rows, 1).float()


def _random_sample(g, G, n, label_lo=0, label_hi=None, size=(0.5, 4.0)):
    W, H = CO.feature_map_size(G['train_cfg'])
    cells = torch.rand(n, 2, generator=g, dtype=torch.float64) * torch.tensor([W, H], dtype=torch.float64)
    hi = sum(G['tasks']) if label_hi is None else label_hi
    return _boxes(g, G, cells, size), torch.randint(label_lo, hi, (n,), generator=g)


def _native(G, boxes, labels, norm_bbox=True):
    from sst_b200 import ops
    cfg = G['train_cfg']
    return ops.centerpoint_targets(torch.cat(boxes).to(dev), torch.cat(labels).to(dev), [b.shape[0] for b in boxes], G['tasks'],
                                   cfg['point_cloud_range'][:2], cfg['voxel_size'][:2], cfg['out_size_factor'], CO.feature_map_size(cfg),
                                   cfg['gaussian_overlap'], cfg['min_radius'], cfg['max_objs'], norm_bbox)


def _check_targets(name, got, ref):
    hm, ab, ind, mask = (list(x) for x in got)
    rhm, rab, rind, rmask = ref
    assert len(hm) == len(rhm)
    for t in range(len(rhm)):
        assert torch.equal(ind[t].cpu(), rind[t]), f"{name} task {t}: ind differs"
        assert torch.equal(mask[t].cpu(), rmask[t]), f"{name} task {t}: mask differs"
        g, r = hm[t].cpu(), rhm[t]
        assert g.shape == r.shape
        assert torch.equal(g != 0, r != 0), f"{name} task {t}: heatmap support differs"
        assert torch.equal(g == 1, r == 1), f"{name} task {t}: heatmap centres differ"
        ulp = (g.view(torch.int32).long() - r.view(torch.int32).long()).abs()
        assert int(ulp.max()) <= 1, f"{name} task {t}: heatmap off by {int(ulp.max())} ulp"
        a = ab[t].cpu()
        assert torch.equal(a[..., [0, 1, 2, 8, 9]], rab[t][..., [0, 1, 2, 8, 9]]), f"{name} task {t}: anno_box offsets / z / velocity"
        assert (a[..., 3:8] - rab[t][..., 3:8]).abs().max().item() <= 1e-6, f"{name} task {t}: anno_box log-dims / sin / cos"


def _radii(G, boxes):
    cfg = G['train_cfg']
    vs, osf = torch.tensor(cfg['voxel_size'][:2]), cfg['out_size_factor']
    b = torch.cat(boxes)
    return CO.gaussian_radius(b[:, 4] / vs[1] / osf, b[:, 3] / vs[0] / osf, cfg['gaussian_overlap'])


SHAPES = {
    "200x136": dict(geom=dict(width=200, height=136), sizes=[150, 0, 60]),
    "136x200": dict(geom=dict(width=136, height=200, tasks=(1, 2), box_dim=9), sizes=[150, 60]),
    "3x200": dict(geom=dict(width=3, height=200), sizes=[40, 10]),
    "150x1": dict(geom=dict(width=150, height=1), sizes=[40]),
    "2x3": dict(geom=dict(width=2, height=3), sizes=[12, 5]),
    "135x201_scalar_zero": dict(geom=dict(width=135, height=201), sizes=[50, 20, 31]),
    "osf1": dict(geom=dict(width=800, height=544), sizes=[120, 40]),
    "osf2": dict(geom=dict(width=400, height=272, out_size_factor=2), sizes=[120, 40]),
    "osf4": dict(geom=dict(width=200, height=136, out_size_factor=4, tasks=(2, 1)), sizes=[120, 40], size=(0.5, 12.0)),
    "osf8": dict(geom=dict(width=100, height=68, out_size_factor=8, box_dim=9), sizes=[120, 40], size=(0.5, 20.0)),
    "overlap0.7": dict(geom=dict(width=200, height=136, gaussian_overlap=0.7), sizes=[150, 60]),
    "min_radius0": dict(geom=dict(width=136, height=200, min_radius=0), sizes=[150, 60], size=(0.05, 1.0)),
    "min_radius40": dict(geom=dict(width=200, height=136, min_radius=40), sizes=[60, 20]),
    "raw_dims_box9": dict(geom=dict(width=200, height=136, tasks=(1, 2), box_dim=9), sizes=[150, 60], norm_bbox=False),
}


@pytest.mark.parametrize("case", list(SHAPES))
def test_targets_map_shapes(case):
    spec = SHAPES[case]
    G = CO.geometry(**spec['geom'])
    g = torch.Generator().manual_seed(list(SHAPES).index(case) + 1)
    samples = [_random_sample(g, G, n, -1, sum(G['tasks']) + 2, spec.get('size', (0.5, 4.0))) for n in spec['sizes']]
    boxes, labels = [s[0] for s in samples], [s[1] for s in samples]
    norm = spec.get('norm_bbox', True)
    W, H = CO.feature_map_size(G['train_cfg'])
    r = _radii(G, boxes)
    if case == "min_radius0":
        assert (r < 1).any(), "no radius-0 box"
    if case == "min_radius40":
        assert r.max().item() < 40
    if case == "135x201_scalar_zero":
        assert len(spec['sizes']) * sum(G['tasks']) * W * H % 2 == 1
    ref = CO.targets(boxes, labels, G['tasks'], G['train_cfg'], norm)
    got = _native(G, boxes, labels, norm)
    _check_targets(case, got, ref)
    assert sum(int(m.sum()) for m in ref[3]) > 0


# ---- slot scan ----
COUNTS = [0, 1, 31, 32, 33, 255, 256, 257, 513]


def _interleaved(counts):
    """labels in round-robin class order while each class has boxes left"""
    left, out = list(counts), []
    while any(left):
        for c in range(len(left)):
            if left[c]:
                out.append(c)
                left[c] -= 1
    return torch.tensor(out, dtype=torch.int64)


def _cut_kind(labels, M):
    """where the max_objs cut falls in the ballot scan: rows (relative to the sample) of the last slot kept and the first cut"""
    rows = torch.cat([torch.where(labels == c)[0] for c in range(len(COUNTS))])
    if M >= rows.numel():
        return "none"
    r1, r2 = int(rows[M - 1]), int(rows[M])
    if labels[r1] != labels[r2]:
        return "class_edge"
    if r1 // 256 != r2 // 256:
        return "chunk_edge" if r2 == r1 + 1 else "chunk"
    if r1 // 32 != r2 // 32:
        return "warp_edge" if r2 == r1 + 1 else "warp"
    return "in_warp"


def _cuts():
    labels = _interleaved(COUNTS)
    cuts = {"m1": 1, "none": labels.numel() + 7}
    for M in range(2, labels.numel()):
        k = _cut_kind(labels, M)
        if k in ("in_warp", "warp_edge", "chunk_edge", "class_edge") and k not in cuts:
            cuts[k] = M
    return cuts


CUTS = _cuts()


def test_slot_cuts_cover_every_kind():
    assert set(CUTS) == {"m1", "none", "in_warp", "warp_edge", "chunk_edge", "class_edge"}
    labels = _interleaved(COUNTS)
    for k, M in CUTS.items():
        if k not in ("m1", "none"):
            assert _cut_kind(labels, M) == k


@pytest.mark.parametrize("cut", list(CUTS))
def test_slot_scan_cuts(cut):
    G = CO.geometry(200, 136, tasks=(len(COUNTS),), max_objs=CUTS[cut])
    g = torch.Generator().manual_seed(7)
    W, H = CO.feature_map_size(G['train_cfg'])
    lab = _interleaved(COUNTS)
    cells = torch.rand(lab.numel(), 2, generator=g, dtype=torch.float64) * torch.tensor([W, H], dtype=torch.float64)
    first = (_boxes(g, G, cells, (0.5, 2.0)), lab)
    second = _random_sample(g, G, 300, -2, len(COUNTS) + 2, (0.5, 2.0))     # starts at row 1378: not on a chunk edge
    boxes, labels = [first[0], second[0]], [first[1], second[1]]
    ref = CO.targets(boxes, labels, G['tasks'], G['train_cfg'])
    _check_targets(f"cut {cut} (max_objs {CUTS[cut]})", _native(G, boxes, labels), ref)
    assert int(ref[3][0][0].sum()) == min(CUTS[cut], lab.numel())


TASKSETS = {"1": (4,), "6": (1, 2, 3, 1, 4, 2), "16": (1, 3, 2, 1, 1, 2, 4, 1, 2, 1, 3, 1, 1, 2, 1, 1)}


def _batch_sizes(name, g):
    if name == "B1":
        return [130]
    if name == "no_boxes":
        return [0, 0, 0]
    B = 33 if name == "B33" else 256
    sizes = torch.randint(1, 40 if B == 33 else 8, (B,), generator=g).tolist()
    sizes[0] = sizes[B // 2] = sizes[-1] = 0
    return sizes


@pytest.mark.parametrize("batch", ["B1", "B33", "B256", "no_boxes"])
@pytest.mark.parametrize("tasks", list(TASKSETS))
def test_slot_tasks_and_batches(tasks, batch):
    G = CO.geometry(48, 40, tasks=TASKSETS[tasks], max_objs=24)
    g = torch.Generator().manual_seed(100 + 7 * list(TASKSETS).index(tasks) + len(batch))
    ncls = sum(G['tasks'])
    samples = [_random_sample(g, G, n, -3, ncls + 3, (0.5, 3.0)) for n in _batch_sizes(batch, g)]
    boxes, labels = [s[0] for s in samples], [s[1] for s in samples]
    ref = CO.targets(boxes, labels, G['tasks'], G['train_cfg'])
    _check_targets(f"{tasks} tasks / {batch}", _native(G, boxes, labels), ref)


def test_slot_limits_raise():
    from sst_b200._lib import SSTB200Error
    g = torch.Generator().manual_seed(3)
    G = CO.geometry(48, 40, tasks=(1,) * 16)
    b, lab = _random_sample(g, G, 30)
    _native(G, [b], [lab])
    with pytest.raises(SSTB200Error):
        _native(CO.geometry(48, 40, tasks=(1,) * 17), [b], [lab])
    G = CO.geometry(48, 40)
    _native(G, [b] + [b[:0]] * 255, [lab] + [lab[:0]] * 255)
    with pytest.raises(SSTB200Error):
        _native(G, [b] + [b[:0]] * 256, [lab] + [lab[:0]] * 256)


# ---- windows ----
CAP = 2 ** 30


def _window_batch():
    G = CO.geometry(60, 36, tasks=(3,))
    W, H = CO.feature_map_size(G['train_cfg'])
    g = torch.Generator().manual_seed(11)
    edge = [(0.01, 0.01), (W - 0.01, 0.01), (0.01, H - 0.01), (W - 0.01, H - 0.01), (W / 2, 0.2), (0.2, H / 2), (W - 0.2, H / 2),
            (W / 2, H - 0.2), (-0.5, 5.3), (7.2, -0.6), (-0.3, -0.4), (W - 0.5, H - 0.5), (W - 1.0, H - 1.0)]
    e = _boxes(g, G, torch.tensor(edge, dtype=torch.float64), (6.0, 14.0))                  # radii past every edge
    cluster = _boxes(g, G, torch.tensor([20.0, 10.0], dtype=torch.float64) + torch.rand(200, 2, generator=g, dtype=torch.float64) *
                     torch.tensor([4.0, 3.0], dtype=torch.float64), (0.5, 5.0))
    cap = _boxes(g, G, torch.tensor([[33.3, 17.6]], dtype=torch.float64))
    cap[0, 3:5] = 4e9                                                                      # radius far above 2^30
    boxes = torch.cat([e, cluster, cap])
    labels = torch.cat([torch.randint(0, 2, (e.shape[0],), generator=g), torch.full((200,), 1), torch.tensor([2])])
    perm = torch.randperm(boxes.shape[0], generator=g)
    return G, [boxes[perm], e[:5]], [labels[perm], torch.tensor([0, 1, 0, 1, 0])]


def test_windows_edges_cluster_and_radius_cap(monkeypatch):
    G, boxes, labels = _window_batch()
    r = _radii(G, boxes)
    assert r.max().item() >= CAP
    draw = CO._draw

    def capped(heatmap, x, y, radius):      # the kernel caps the radius at 2^30: exp(-d^2 / 2 sigma^2) rounds to 1 over the whole map
        if radius >= CAP:
            heatmap.fill_(1.0)
        else:
            draw(heatmap, x, y, radius)
    monkeypatch.setattr(CO, "_draw", capped)
    ref = CO.targets(boxes, labels, G['tasks'], G['train_cfg'])
    a = _native(G, boxes, labels)
    b = _native(G, boxes, labels)
    for u, v in zip(a, b):
        for s, w in zip(u, v):
            assert s.cpu().numpy().tobytes() == w.cpu().numpy().tobytes(), "two runs differ"
    _check_targets("windows", a, ref)
    assert torch.equal(a[0][0][0, 2].cpu(), torch.ones_like(a[0][0][0, 2].cpu()))
    assert (a[0][0][0, :2] != 0).sum().item() > 0 and (a[0][0][0, :2] < 1).any()


# ---- dirty outputs through the C ABI ----
def test_targets_rewrite_dirty_outputs_c_abi():
    from sst_b200 import _lib
    G = CO.geometry(135, 201, tasks=(1, 4, 4), box_dim=9, max_objs=70)
    cfg = G['train_cfg']
    W, H = CO.feature_map_size(cfg)
    g = torch.Generator().manual_seed(5)
    sizes = [60, 0, 45]
    samples = [_random_sample(g, G, n, -1, 11) for n in sizes]
    boxes, labels = [s[0] for s in samples], [s[1] for s in samples]
    B, M = len(sizes), cfg['max_objs']
    # task 0: B ncls H W odd -> scalar zeroing; task 1: a multiple of 4, aligned -> float4; task 2: the same size one float off -> scalar
    n = [B * c * H * W for c in G['tasks']]
    assert n[0] % 2 == 1 and n[1] % 4 == 0
    hm_buf = [torch.full((n[0],), float('nan'), device=dev), torch.full((n[1],), float('nan'), device=dev),
              torch.full((n[2] + 1,), float('nan'), device=dev)]
    hm_ptr = [hm_buf[0].data_ptr(), hm_buf[1].data_ptr(), hm_buf[2].data_ptr() + 4]
    ab = [torch.full((B, M, 10), float('nan'), device=dev) for _ in G['tasks']]
    ind = [torch.full((B, M), -1, dtype=torch.int64, device=dev) for _ in G['tasks']]
    mask = [torch.full((B, M), 255, dtype=torch.uint8, device=dev) for _ in G['tasks']]
    bx, lb = torch.cat(boxes).to(dev), torch.cat(labels).to(dev)
    pp = lambda ps: (C.c_void_p * len(ps))(*ps)
    task_off = np.cumsum([0] + list(G['tasks'])).tolist()
    c = _lib.ctx(dev)
    rc = _lib.lib().sstb200_centerpoint_targets(
        c, bx.data_ptr(), lb.data_ptr(), 9, _lib.arr(C.c_int32, np.cumsum([0] + sizes).tolist()), B, _lib.arr(C.c_int32, task_off),
        len(G['tasks']), _lib.arr(C.c_float, cfg['point_cloud_range'][:2]), _lib.arr(C.c_float, list(cfg['voxel_size'][:2])), 1, W, H,
        cfg['gaussian_overlap'], cfg['min_radius'], M, 1, pp(hm_ptr), pp([t.data_ptr() for t in ab]), pp([t.data_ptr() for t in ind]),
        pp([t.data_ptr() for t in mask]))
    assert rc == 0
    torch.cuda.synchronize()
    hm = [hm_buf[0].view(B, 1, H, W), hm_buf[1].view(B, 4, H, W), hm_buf[2][1:].view(B, 4, H, W)]
    assert torch.isnan(hm_buf[2][0]).item(), "the float before the offset heatmap was written"
    ref = CO.targets(boxes, labels, G['tasks'], cfg)
    _check_targets("dirty", (hm, ab, ind, mask), ref)


# ---------------------------------------------------------------------------------------------------------------------------------------
# Gaussian focal loss
# ---------------------------------------------------------------------------------------------------------------------------------------
def _G(s, t):
    """float64 d loss / d logit of one element at sigmoid s, without the clamp"""
    q, u4 = 1 - s, (1 - t) ** 4
    d = (s * s / (q + 1e-12) - 2 * s * torch.log(q + 1e-12)) * u4
    d = d + torch.where(t == 1, -q * q / (s + 1e-12) + 2 * q * torch.log(s + 1e-12), torch.zeros_like(s))
    return d * s * q


def _fl_err_unit(x64, t64):
    """the first-order fp32 error of the kernel's per-element gradient (before the scale; _check_fl_grad adds the subnormal
    spacing)"""
    s = torch.sigmoid(x64)
    q, u4 = 1 - s, (1 - t64) ** 4
    g0 = _G(s, t64)
    d = 2.0 ** -21
    env = torch.maximum((_G(s * (1 + d), t64) - g0).abs(), (_G(s * (1 - d), t64) - g0).abs())
    terms = u4 * (s ** 3 + 2 * s * s * q * torch.log(q + 1e-12).abs())
    terms = terms + torch.where(t64 == 1, q ** 3 + 2 * s * q * q * torch.log(s + 1e-12).abs(), torch.zeros_like(s))
    logq = torch.where(q >= 0.5, u4 * 2 * s * s * 2.0 ** -25, torch.zeros_like(s))
    return torch.nan_to_num(env + terms * 2.0 ** -20 + logq, nan=0.0)


def _fl_loss_err(x64, t64):
    """the first-order fp32 error of the kernel's per-element loss: the sigmoid's relative error 2^-21 pushed through the loss, 2^-20
    of each term and the rounding of 1 - p (2^-25 absolute for p <= 1/2) pushed through log(1 - p)"""
    u4 = (1 - t64) ** 4

    def loss(p):
        q = 1 - p
        return -torch.log(q + 1e-12) * p * p * u4 + torch.where(t64 == 1, -torch.log(p + 1e-12) * q * q, torch.zeros_like(p))
    p = torch.sigmoid(x64).clamp(LO, HI)
    l0, d = loss(p), 2.0 ** -21
    env = torch.maximum((loss(p * (1 + d)) - l0).abs(), (loss(p * (1 - d)) - l0).abs())
    logq = torch.where(p <= 0.5, p * p * u4 * 2.0 ** -25 / (1 - p), torch.zeros_like(p))
    return torch.nan_to_num(env + l0.abs() * 2.0 ** -20 + logq, nan=0.0)


def _check_fl_loss(name, loss, ref, x, t, loss_weight, num_pos):
    """the loss against the oracle's within LOSS_C times its elements' summed first-order error (and the final fp32 rounding);
    returns the error in those units"""
    unit = loss_weight * float(_fl_loss_err(x.double(), t.double()).sum()) / max(num_pos, 1.0) + abs(ref) * 2.0 ** -24
    err = abs(loss - ref)
    assert err <= LOSS_C * unit, f"{name}: loss {loss} against {ref}: {err / unit:.3g} units"
    return err / unit


def _kernel_sigmoid_hi(x64):
    """the kernel's fp32 sigmoid 1 / (1 + expf(-x)) where the arithmetic fixes it (1 + e more than 1% of an fp32 step from a rounding
    tie, so expf's 2 ulp cannot move it), else NaN; only for e < 1"""
    e = torch.exp(-x64)
    k = e * 2.0 ** 23
    frac = k - torch.floor(k)
    fixed = ((frac - 0.5).abs() > 0.01) & (e < 1)
    v = (1 + torch.round(k) * 2.0 ** -23).float()
    s = (torch.ones_like(v) / v).double()
    return torch.where(fixed, s, torch.full_like(s, float('nan')))


def _check_fl_grad(name, got, x, t, ref, scale):
    """per-element check of the focal gradient; returns the worst error in units of the first-order bound"""
    x64, t64 = x.double(), t.double()
    got = got.cpu().double()
    nan = torch.isnan(x64)
    assert torch.equal(torch.isnan(got), nan), f"{name}: NaN gradients at {int((torch.isnan(got) != nan).sum())} wrong elements"
    s = torch.sigmoid(x64)
    unit = _fl_err_unit(x64, t64) * abs(scale) + 2.0 ** -149 * (1 + abs(scale))
    unclamped = _G(s, t64) * scale
    band = ((s - LO).abs() <= FL_BAND * ULP_LO) | ((s - HI).abs() <= FL_BAND * ULP_HI)
    outside = ~band & ~nan
    err = (got - ref).abs()
    clamped = outside & ((s < LO) | (s > HI))
    passed = outside & ~clamped
    assert (got[clamped] == 0).all(), f"{name}: {int((got[clamped] != 0).sum())} clamped elements with a gradient"
    bad = passed & (err > FL_GRAD_C * unit)
    assert not bad.any(), f"{name}: {int(bad.sum())} elements off, worst {float((err / unit)[bad].max()):.3g} e"
    inb = band & ~nan
    ok = (got[inb] == 0) | ((got[inb] - unclamped[inb]).abs() <= FL_GRAD_C * unit[inb])
    assert ok.all(), f"{name}: {int((~ok).sum())} in-band elements neither 0 nor the unclamped value"
    s32 = _kernel_sigmoid_hi(x64)
    fixed = inb & ~torch.isnan(s32) & (s > 0.5)
    if fixed.any():
        want_pass = s32[fixed] <= float(np.float32(HI))
        g = got[fixed]
        assert torch.equal(g != 0, want_pass | (unclamped[fixed] == 0)), f"{name}: the fp32 inclusive clamp at 0.9999f is not followed"
    ratio = (err / unit)[passed & (unit > 0)]
    return float(ratio.max()) if ratio.numel() else 0.0


def _fl_data(n, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g) * 4 - 2
    t = torch.rand(n, generator=g) ** 4
    pick = torch.rand(n, generator=g)
    t[pick < 0.4] = 0.0
    t[(pick >= 0.4) & (pick < 0.42)] = 1.0
    t[(pick >= 0.42) & (pick < 0.43)] = float(np.nextafter(np.float32(1), np.float32(0)))
    t[(pick >= 0.43) & (pick < 0.44)] = 1e-30
    t[0] = 1.0
    if n > 3:
        x[1], x[2] = float('inf'), -float('inf')
    return x, t


def _fl_run(x, t, loss_weight=1.0, upstream=1.0, half=False):
    """(native loss, num_pos, grad), (oracle loss, num_pos, grad)"""
    from sst_b200 import ops
    xin = x.half() if half else x
    x64 = xin.double().requires_grad_(True)
    ref, num_pos = CO.focal_loss(x64, t.double(), loss_weight)
    ref.backward(torch.tensor(upstream, dtype=torch.float64))
    xg = xin.to(dev).requires_grad_(True)
    loss, npos = ops.gaussian_focal_loss(xg, t.to(dev), loss_weight)
    loss.backward(torch.tensor(upstream, device=dev))
    assert xg.grad.dtype == xin.dtype
    return (loss.item(), npos.item(), xg.grad), (ref.item(), num_pos, x64.grad), upstream * loss_weight / max(num_pos, 1.0)


def _fl_sizes():
    S = torch.cuda.get_device_properties(dev).multi_processor_count if torch.cuda.is_available() else 132
    N = 8 * 2048 * S
    return [1, 255, 256, 257, 2047, 2048, 2049, N - 1, N, N + 1, 3 * N + 5]


@pytest.mark.parametrize("k", range(11))
def test_focal_grid_sizes(k):
    n = _fl_sizes()[k]
    x, t = _fl_data(n, 40 + k)
    (loss, npos, grad), (ref, num_pos, rgrad), scale = _fl_run(x, t)
    assert npos == num_pos
    lerr = _check_fl_loss(f"n={n}", loss, ref, x, t, 1.0, num_pos)
    worst = _check_fl_grad(f"n={n}", grad, x, t, rgrad, scale)
    print(f"focal n={n}: loss {lerr:.3f} units (rel {abs(loss - ref) / abs(ref):.2e}), gradient worst {worst:.3f} e")


def _sweep_logits():
    """fp32 logits around both clamp bounds: at logit(1e-4) one logit ulp at a time, at logit(0.9999f) the fp32 values nearest to each
    of +-64 sigmoid ulps; plus, at the upper bound, logits whose kernel sigmoid is exactly 0.9999f and its two neighbours"""
    lo = np.array([math.log(LO / (1 - LO))], dtype=np.float32).view(np.int32)[0]
    low = (np.arange(-64, 65, dtype=np.int32) + lo).view(np.float32)
    hi32 = float(np.float32(HI))
    high = np.array([math.log(s / (1 - s)) for s in (hi32 + k * ULP_HI for k in range(-64, 65))], dtype=np.float32)
    exact = []
    for k in (838, 839, 840):       # 1 + e = 1 + k 2^-23: 1 / (1 + 839 2^-23) rounds to 0.9999f exactly
        e = k * 2.0 ** -23
        exact += [-math.log(e * (1 + f * 2.0 ** -24 / e)) for f in (-0.25, 0.0, 0.25)]
    return torch.from_numpy(np.concatenate([low, high, np.array(exact, dtype=np.float32)]))


def test_focal_clamp_bounds():
    xs = _sweep_logits()
    x = xs.repeat(4)
    t = torch.cat([torch.full_like(xs, v) for v in (0.0, 0.5, 1.0, float(np.nextafter(np.float32(1), np.float32(0))))])
    (loss, npos, grad), (ref, num_pos, rgrad), scale = _fl_run(x, t)
    assert npos == num_pos
    lerr = _check_fl_loss("clamp sweep", loss, ref, x, t, 1.0, num_pos)
    worst = _check_fl_grad("clamp sweep", grad, x, t, rgrad, scale)
    s = torch.sigmoid(x.double())
    for b, u in ((LO, ULP_LO), (HI, ULP_HI)):
        d = (s - b) / u
        assert (d < -FL_BAND).any() and (d > FL_BAND).any() and (d.abs() <= FL_BAND).any()
    s32 = _kernel_sigmoid_hi(x.double())
    assert (s32 == float(np.float32(HI))).sum() >= 3, "no logit whose kernel sigmoid is exactly 0.9999f"
    print(f"focal clamp sweep: loss {lerr:.3f} units (rel {abs(loss - ref) / abs(ref):.2e}), gradient worst {worst:.3f} e")


def test_focal_nan_logits():
    x, t = _fl_data(5000, 77)
    x[[10, 999, 4999]] = float('nan')
    t[999] = 1.0
    (loss, npos, grad), (ref, num_pos, rgrad), scale = _fl_run(x, t)
    assert math.isnan(ref) and math.isnan(loss), f"loss {loss} for NaN logits"
    assert npos == num_pos
    keep = ~torch.isnan(x)
    _check_fl_grad("NaN logits", grad, x, t, torch.where(keep, rgrad, torch.full_like(rgrad, float('nan'))), scale)


@pytest.mark.parametrize("variant", ["loss_weight", "upstream_2^16", "fp16"])
def test_focal_scaling_and_fp16(variant):
    x, t = _fl_data(300000, 91)
    kw = dict(loss_weight=1.5) if variant == "loss_weight" else dict(upstream=65536.0) if variant == "upstream_2^16" else dict(half=True)
    (loss, npos, grad), (ref, num_pos, rgrad), scale = _fl_run(x, t, **kw)
    assert npos == num_pos
    lerr = _check_fl_loss(variant, loss, ref, x.half().float() if variant == "fp16" else x, t, kw.get('loss_weight', 1.0), num_pos)
    print(f"focal {variant}: loss {lerr:.3f} units")
    if variant == "fp16":
        xh = x.half().float()
        g = grad.cpu().double()
        # the gradient as the fp32 kernel gives it, then rounded to fp16 (half an fp16 ulp, subnormals included)
        bound = FL_GRAD_C * _fl_err_unit(xh.double(), t.double()) * scale + rgrad.abs() * 2.0 ** -11 + 2.0 ** -25
        s = torch.sigmoid(xh.double())
        inside = ((s - LO).abs() > FL_BAND * ULP_LO) & ((s - HI).abs() > FL_BAND * ULP_HI)
        assert ((g - rgrad).abs() <= bound)[inside].all()
    else:
        _check_fl_grad(variant, grad, x, t, rgrad, scale)


# ---------------------------------------------------------------------------------------------------------------------------------------
# L1 loss
# ---------------------------------------------------------------------------------------------------------------------------------------
def _l1_inputs(seed, B, M, W, H, mask_p=0.7, nan_p=0.0, cw=None):
    g = torch.Generator().manual_seed(seed)
    preds = {k: torch.randn(B, c, H, W, generator=g) for k, c in (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))}
    ab = torch.randn(B, M, 10, generator=g)
    if nan_p:
        ab[torch.rand(B, M, 10, generator=g) < nan_p] = float('nan')
    ind = torch.randint(0, H * W, (B, M), generator=g)
    ind[:, 0] = 0
    if M > 1:
        ind[:, -1] = H * W - 1
    mask = (torch.rand(B, M, generator=g) < mask_p).to(torch.uint8)
    mask[:, 0] = 1
    cw = cw or [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2, 0.0, 0.5]
    return preds, ab, ind, mask, cw


def _l1_abs_sum(preds, ab, ind, mask, cw, lw, upstream):
    """float64 per element: the sum over the slots gathering it of |d loss / d pred|, and the number of those slots (the kernel's
    rounding: g = gl lw / avg and each g w in fp32, then a sequential fp32 sum)"""
    B, M = ind.shape
    p = torch.cat([preds[k] for k, _ in (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))], 1).double()
    C_, H, W = p.shape[1:]
    avg = float(mask.float().sum() + 1e-4)
    w = mask.double()[..., None] * (~torch.isnan(ab)).double() * torch.tensor(cw, dtype=torch.float32).double()
    pg = p.permute(0, 2, 3, 1).reshape(B, H * W, C_).gather(1, ind[..., None].expand(B, M, C_))
    contrib = w * (pg - ab.double()).sign().abs().nan_to_num(0.0) * abs(upstream * lw / avg)
    out = []
    for v in (contrib, (contrib > 0).double()):
        o = torch.zeros(B, H * W, C_, dtype=torch.float64)
        o.scatter_add_(1, ind[..., None].expand(B, M, C_), v)
        out.append(dict(zip(("reg", "height", "dim", "rot", "vel"), o.view(B, H, W, C_).permute(0, 3, 1, 2).split([2, 1, 3, 2, 2], 1))))
    return out


def _l1_run(preds, ab, ind, mask, cw, lw=2.0, upstream=1.0):
    from sst_b200 import ops
    p64 = {k: v.double().requires_grad_(True) for k, v in preds.items()}
    ref = CO.l1_loss(p64, ab, ind, mask, cw, lw)
    ref.backward(torch.tensor(upstream, dtype=torch.float64))
    pg = {k: v.to(dev).requires_grad_(True) for k, v in preds.items()}
    loss = ops.centerpoint_l1_loss(pg, ab.to(dev), ind.to(dev), mask.to(dev), cw, lw)
    loss.backward(torch.tensor(upstream, device=dev))
    return loss.item(), ref.item(), {k: v.grad for k, v in pg.items()}, {k: v.grad for k, v in p64.items()}


def _check_l1(name, preds, ab, ind, mask, cw, lw=2.0, upstream=1.0):
    loss, ref, grads, rgrads = _l1_run(preds, ab, ind, mask, cw, lw, upstream)
    if math.isnan(ref):
        assert math.isnan(loss), f"{name}: loss {loss}, the oracle's is NaN"
        rel = 0.0
    else:
        rel = abs(loss - ref) / max(abs(ref), 1e-30)
        assert rel <= L1_RTOL or loss == ref, f"{name}: loss rel err {rel:.2e}"
    absum, count = _l1_abs_sum(preds, ab, ind, mask, cw, lw, upstream)
    worst = 0.0
    for k in grads:
        g, r, a = grads[k].cpu().double(), rgrads[k], absum[k]
        assert not torch.isnan(g).any() and not torch.isnan(r).any(), f"{name} {k}: NaN gradient"
        assert (g[a == 0] == 0).all() and (r[a == 0] == 0).all(), f"{name} {k}: a gradient where no slot contributes"
        err = (g - r).abs()
        unit = a * (count[k] + 2) * 2.0 ** -24      # two roundings of g w, one per term of the sum
        assert (err <= L1_GRAD_C * unit).all(), f"{name} {k}: gradient off by {float((err / unit.clamp_min(1e-300)).max()):.3g} units"
        if (unit > 0).any():
            worst = max(worst, float((err / unit)[unit > 0].max()))
    print(f"L1 {name}: loss rel err {rel:.2e}, gradient worst {worst:.3f} units")
    return grads


L1_SIZES = [(1, 1, 53, 37), (255, 17, 37, 53), (256, 5, 53, 37), (257, 17, 37, 53), (4096, 3, 53, 37)]


@pytest.mark.parametrize("M,B,W,H", L1_SIZES, ids=[f"M{m}_B{b}_{w}x{h}" for m, b, w, h in L1_SIZES])
def test_l1_sizes(M, B, W, H):
    preds, ab, ind, mask, cw = _l1_inputs(M + B, B, M, W, H, nan_p=0.02)
    _check_l1(f"M={M} B={B}", preds, ab, ind, mask, cw)
    preds, ab, ind, mask, cw = _l1_inputs(M + B + 1, B, M, W, H, cw=[1.0] * 10)
    _check_l1(f"M={M} B={B} finite", preds, ab, ind, mask, cw, lw=0.25, upstream=65536.0)


def test_l1_limits():
    from sst_b200._lib import SSTB200Error
    preds, ab, ind, mask, cw = _l1_inputs(1, 1, 4097, 20, 10)
    with pytest.raises(SSTB200Error):
        _l1_run(preds, ab, ind, mask, cw)


def test_l1_every_mask_zero():
    preds, ab, ind, mask, cw = _l1_inputs(2, 3, 300, 37, 53)
    mask.zero_()
    loss, ref, grads, _ = _l1_run(preds, ab, ind, mask, cw)
    assert loss == 0.0 and ref == 0.0
    for g in grads.values():
        assert not g.any()


def test_l1_shared_cells_sum_in_slot_order():
    """one cell shared by slots 0, 255, 256 and 300 (across the backward's 256-slot passes) and twenty cells each shared by slots
    260 + i, 516 + i and 3000 + i (none below 256): each cell's gradient is its slots' sum, and two runs are bit-identical"""
    preds, ab, ind, mask, cw = _l1_inputs(9, 2, 4096, 53, 37, mask_p=0.0, cw=[1.0] * 10)
    ind.random_(1, 53 * 37 - 1, generator=torch.Generator().manual_seed(1))
    for s in (0, 255, 256, 300):
        ind[:, s], mask[:, s] = 1234, 1
    for i in range(20):
        for s in (260 + i, 516 + i, 3000 + i):
            ind[:, s], mask[:, s] = 100 + i, 1
    ab[:, :, :] = -10.0            # every sign +1: the sums do not cancel
    runs = [_check_l1("shared cells", preds, ab, ind, mask, cw) for _ in range(2)]
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k])
        assert (runs[0][k][:, :, 1234 // 53, 1234 % 53] > 0).all()


def test_l1_nan_prediction_at_masked_out_slot():
    """the reference gathers every slot and weights a masked-out one by 0: a NaN prediction at its cell makes the loss NaN; one at a
    cell no slot gathers does not"""
    preds, ab, ind, mask, cw = _l1_inputs(12, 2, 40, 37, 53)
    ind[1, 7], mask[1, 7] = 500, 0
    assert not ((ind == 500) & (mask == 1)).any()
    gathered = set(ind.flatten().tolist())
    free = next(c for c in range(37 * 53) if c not in gathered)
    preds['dim'][1, 2].view(-1)[free] = float('nan')
    loss, ref, _, _ = _l1_run(preds, ab, ind, mask, cw)
    assert math.isfinite(loss) and math.isfinite(ref)
    preds['dim'][1, 2].view(-1)[500] = float('nan')
    _check_l1("NaN prediction, masked-out slot", preds, ab, ind, mask, cw)


def test_l1_nan_targets_and_zero_code_weights():
    preds, ab, ind, mask, _ = _l1_inputs(13, 4, 200, 53, 37)
    ab[0, 0, 3] = float('nan')                         # a masked slot: NaN loss, no gradient from it
    cw = [1.0, 0.0, 1.0, 0.0, 1.0, 1.0, 0.0, 1.0, 0.0, 0.0]
    grads = _check_l1("NaN target, zero code weights", preds, ab, ind, mask, cw)
    assert not grads['reg'][:, 1].any() and not grads['vel'].any()


# ---------------------------------------------------------------------------------------------------------------------------------------
# module level
# ---------------------------------------------------------------------------------------------------------------------------------------
MODULE_GEOM = dict(width=200, height=136, out_size_factor=2, voxel_size=(0.2, 0.2), tasks=(1, 2), box_dim=9)


def test_center_head_loss_nonsquare():
    import sst_b200  # noqa: F401
    from sst_b200.centerhead_modules import CenterHead
    G = CO.geometry(**MODULE_GEOM)
    head = CenterHead(**{k: v for k, v in CO.head_cfg(G).items() if k != 'type'})
    raw, labels = CO.synth_batch(8, G, [90, 0, 40])
    preds = CO.synth_preds(8, G, 3)
    leaves = [[{k: v.to(dev).requires_grad_(True) for k, v in pd[0].items()}] for pd in preds]
    losses = head.loss([b.to(dev) for b in raw], [l.to(dev) for l in labels], leaves)
    sum(losses.values()).backward()
    hm, ab, ind, mask = CO.targets([CO.gravity(b) for b in raw], labels, G['tasks'], G['train_cfg'])
    for t, pd in enumerate(preds):
        p64 = {k: v.double().requires_grad_(True) for k, v in pd[0].items()}
        lh, _ = CO.focal_loss(p64['heatmap'], hm[t].double())
        lb = CO.l1_loss(p64, ab[t], ind[t], mask[t], G['train_cfg']['code_weights'], G['loss_bbox_weight'])
        (lh + lb).backward()
        for name, ref in ((f"task{t}.loss_heatmap", lh), (f"task{t}.loss_bbox", lb)):
            assert abs(losses[name].item() - ref.item()) <= 1e-5 * abs(ref.item()), name
        for k, v in p64.items():
            g = leaves[t][0][k].grad.cpu().double()
            assert (g - v.grad).abs().max().item() <= 1e-4 * v.grad.abs().max().item() + 1e-30, f"task {t} {k}"


def _sparse_preds(G, seed, batch, n):
    """heatmap logits -12 except at n well-separated cells per sample with distinct logits; small boxes there"""
    W, H = CO.feature_map_size(G['train_cfg'])
    g = torch.Generator().manual_seed(seed)
    preds = CO.synth_preds(seed, G, batch, scale=0.3)
    logit = 0.0
    for pd in preds:
        p = pd[0]
        p['heatmap'].fill_(-12.0)
        p['dim'] = torch.randn(p['dim'].shape, generator=g) * 0.2 - 1.0
        for b in range(batch):
            for k, cell in enumerate(torch.randperm((H // 4) * (W // 4), generator=g)[:n].tolist()):
                logit += 1e-3
                p['heatmap'][b, k % p['heatmap'].shape[1], 4 * (cell // (W // 4)), 4 * (cell % (W // 4))] = -1.5 + logit
    return preds


def test_get_bboxes_nonsquare():
    import sst_b200  # noqa: F401
    from sst_b200.centerhead_modules import CenterHead
    G = CO.geometry(**MODULE_GEOM)
    preds = _sparse_preds(G, 31, 2, 60)
    ref = CO.get_bboxes(preds, G['tasks'], G['bbox_coder'], G['test_cfg'])
    for pd in preds:     # no BEV IoU among a task's candidates lies within 1e-4 of nms_thr
        for c in CO.decode(pd[0]['heatmap'].sigmoid(), pd[0]['rot'][:, 0:1], pd[0]['rot'][:, 1:2], pd[0]['height'], pd[0]['dim'].exp(),
                           pd[0]['vel'], pd[0]['reg'], G['bbox_coder']):
            keep = c['scores'] >= G['test_cfg']['score_threshold']
            bev = CO.bev_xyxyr(c['bboxes'][keep])
            assert IO.drop_near_threshold(bev, [G['test_cfg']['nms_thr']]).numel() == bev.shape[0]
    head = CenterHead(**{k: v for k, v in CO.head_cfg(G).items() if k != 'type'})
    got = head.get_bboxes([[{k: v.to(dev) for k, v in pd[0].items()}] for pd in preds], [dict() for _ in range(2)])
    for (gb, gs, gl), (rb, rs, rl) in zip(got, ref):
        assert gb.shape == rb.shape and rb.shape[0] > 0
        assert torch.equal(gl.cpu(), rl)
        assert (gs.cpu() - rs).abs().max().item() <= 1e-6
        assert (gb.cpu() - rb).abs().max().item() <= 1e-4
