"""GPU: the fused voxel feature encoder (csrc/vfe.cu: DynamicVFE, DynamicScatterVFE) against float64 on every dispatch route,
tile edge and dirty workspace.

`vfe_forward_impl` picks one of four routes:
    tile, fp32   mode max, (C0, C1) in (64,128) (64,64) (64,0) (32,64): layer 0 in 128-point tiles (segmented max, atomicMax on
                 the float bits across row groups and tiles), layer 1 in vfe_fused_kernel phase 1
    tile, bf16   the same with precision "bf16" and C1 > 0: layer 1 on wgmma (bf16 operands, fp32 accumulate)
    fused        every other instantiated pair and all of mode avg: one warp per voxel
    wide         D0 = F + 3 cluster + 3 centre > 16 (or F > 32): decorated rows, row GEMMs, segment reduce
Each route is run for both classes (int32 coordinates with the drop-first rule of DynamicScatter, int64 without; test_routes
walks the table), on CSR layouts that put voxel boundaries on and across the 16 / 32 / 64-row groups and the 128-row tiles, on a
voxel spanning three tiles, on 1 / 127 / 128 / 129 valid points and on more points than the persistent tile loops cover in one pass.  Every feature run goes through
the C entry point with a workspace left full of large values by a previous call and an output buffer prefilled with a sentinel
that rows beyond the voxel count must keep.  DynamicVFE's drop-first rule removes a sample's (-1,-1,-1) row when the sample has
a point with a negative coordinate, and its first voxel otherwise (test_batch_dynamic_vfe).

Reference: oracle.sst_oracle.dynamic_vfe_forward / dynamic_scatter_vfe_forward on float64 points, weights and BatchNorm buffers.
Both sides get the same float32-rounded voxel size, and the grid ratios are integers, so the oracle's round() canvas and the
module's float32 ceil canvas agree (the centre offsets differ by one float32 rounding, well inside the bound).  Voxel coordinates, the inverse and the voxel count are compared bit-exactly.

Error metric: besides a max-norm check, every comparison asserts a PER-VOXEL-ROW bound
    |out[v] - ref[v]|_inf  <=  tol * |mag[v]|_inf
where mag is the float64 magnitude propagated through the encoder: a decorated feature that is a difference gets the sum of its
operands' magnitudes ((|x| + |mean|) / scaler for the cluster term, |x| + |c v| + |offset| for the centre term, which keeps the
cancellation near |x| = 75 m from tripping an fp32 tolerance), then per layer |X| @ |W|^T * |s| + |beta| + |running_mean s|, pooled
with a max, and [mag0 || pooled mag0] for layer 1.  Tolerances: fp32 1e-5; bf16 layer 1 5e-3 (two bf16 operand roundings give at
most 2^-8 relative per product).  Max-norm, relative to the largest reference value: fp32 1e-4, bf16 1e-2."""
import copy
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

F32 = lambda v: float(np.float32(v))  # noqa: E731
VS = (F32(0.32), F32(0.32), F32(0.2))
RNG = (-74.88, -74.88, -2.0, 74.88, 74.88, 4.0)  # 468 x 468 x 30 cells
GRID_ZYX = (30, 468, 468)
ROW_TOL = {"fp32": 1e-5, "bf16": 5e-3}
MAX_TOL = {"fp32": 1e-4, "bf16": 1e-2}
EPS = 1e-3
SENTINEL = 1e30
POISON = 1e4

TILE = ((64, 128), (64, 64), (64, 0), (32, 64))
TILE_L1 = ((64, 128), (64, 64), (32, 64))  # tile pairs whose layer 1 runs on wgmma with precision "bf16"
FUSED = ((64, 128), (64, 64), (32, 64), (64, 0), (128, 128), (128, 0), (32, 0), (32, 32), (64, 256))

# CSR layouts (point counts per output voxel, in (b, z, y, x) order).  EDGE_A ends voxels exactly at rows 15|16, 16|17, 31|32,
# 63|64, 127|128 and 128|129 and is padded to two full tiles; EDGE_B has a voxel straddling each of those edges.
EDGE_A = [5, 11, 1, 15, 20, 12, 30, 34, 1, 7, 3, 2, 1, 1, 9, 40, 64]
EDGE_B = [14, 5, 11, 4, 28, 4, 60, 5, 2, 1, 6]
assert np.cumsum(EDGE_A)[[1, 2, 3, 5, 7, 8]].tolist() == [16, 17, 32, 64, 128, 129] and sum(EDGE_A) == 256
assert np.cumsum(EDGE_B)[[0, 1, 5, 6, 7]].tolist() == [14, 19, 66, 126, 131]


def _random_counts(seed, total, hi):
    g = np.random.default_rng(seed)
    out = []
    while sum(out) < total:
        out.append(int(g.integers(1, hi + 1)))
    out[-1] -= sum(out) - total
    return [c for c in out if c > 0]


@functools.lru_cache(maxsize=None)
def _persistent_total():
    """more valid points than one pass of the persistent tile loops (grid 3 * SMs CTAs of 128 points)"""
    return 3 * torch.cuda.get_device_properties(0).multi_processor_count * 128 + 3001


def _layout(name):
    """per-sample lists of voxel point counts"""
    if name == "edges":
        return [EDGE_A + EDGE_B, _random_counts(5, 600, 40)]
    if name == "one_point":
        return [[1]]
    if name == "big_voxel":  # rows 7 .. 336: three tiles
        return [[7, 330, 5]]
    if name.startswith("total_"):
        return [_random_counts(int(name[6:]), int(name[6:]), 9)]
    if name == "persistent":
        return [_random_counts(11, _persistent_total(), 12)]
    raise ValueError(name)


# ----------------------------------------------------------------------------------------------------------------------
# data, module, float64 reference
# ----------------------------------------------------------------------------------------------------------------------
def _cloud(counts, F, seed, drop_first, invalid=None):
    """points [P, F] fp32 and coordinates [P, 4] (b, z, y, x) int64 with the given voxel counts per sample, rows shuffled.
    drop_first: every non-empty sample gets an extra first voxel (3 points) that DynamicScatter's rule removes, unless the sample
    has invalid points.  invalid: {sample: n} points with coordinates (b, -1, -1, -1)."""
    invalid = invalid or {}
    g = torch.Generator().manual_seed(seed)
    pts, cos = [], []
    vs = torch.tensor(VS, dtype=torch.float64)
    lo = torch.tensor(RNG[:3], dtype=torch.float64)
    ncell = GRID_ZYX[0] * GRID_ZYX[1] * GRID_ZYX[2]
    for b, cnt in enumerate(counts):
        cnt = list(cnt)
        if drop_first and cnt and not invalid.get(b):
            cnt = [3] + cnt
        if cnt:
            cand = torch.unique(torch.randint(0, ncell, (2 * len(cnt) + 8,), generator=g))
            cells = torch.sort(cand[torch.randperm(cand.numel(), generator=g)[:len(cnt)]]).values
            assert cells.numel() == len(cnt)
            zyx = torch.stack([cells // (GRID_ZYX[1] * GRID_ZYX[2]), cells // GRID_ZYX[2] % GRID_ZYX[1], cells % GRID_ZYX[2]], 1)
            zyx = zyx.repeat_interleave(torch.tensor(cnt), 0)
            xyz = (zyx.flip(1).double() + torch.rand((zyx.shape[0], 3), generator=g, dtype=torch.float64)) * vs + lo
            pts.append(torch.cat([xyz, torch.randn((zyx.shape[0], F - 3), generator=g, dtype=torch.float64) * 2], 1).float())
            cos.append(torch.cat([torch.full((zyx.shape[0], 1), b, dtype=torch.int64), zyx], 1))
        n = invalid.get(b, 0)
        if n:
            pts.append((torch.randn((n, F), generator=g) * 30).float())
            cos.append(torch.tensor([[b, -1, -1, -1]], dtype=torch.int64).repeat(n, 1))
    pts, co = torch.cat(pts), torch.cat(cos)
    perm = torch.randperm(pts.shape[0], generator=g)
    pts, co = pts[perm], co[perm]
    last = int(torch.nonzero(co[:, 0] == co[:, 0].max())[0])  # the batch size is read from the last row
    order = torch.cat([torch.arange(last), torch.arange(last + 1, pts.shape[0]), torch.tensor([last])])
    return pts[order].contiguous(), co[order].contiguous()


def _module(cls, F, C0, C1, mode, cluster=True, centre=True, seed=0, scaler=10.0):
    """the module with non-trivial BatchNorm (random running statistics, gamma of both signs, nonzero beta) and, per layer, one
    channel that the ReLU always clears and one that is always active"""
    from sst_b200.voxel_modules import DynamicScatterVFE, DynamicVFE
    norm = dict(type="BN1d", eps=EPS, momentum=0.01)
    kw = dict(in_channels=F, feat_channels=[C0] + ([C1] if C1 else []), with_cluster_center=cluster, with_voxel_center=centre,
              voxel_size=VS, point_cloud_range=RNG, norm_cfg=norm, mode=mode)
    if cls == "scatter":
        kw["rel_dist_scaler"] = scaler
    torch.manual_seed(seed)
    m = (DynamicScatterVFE if cls == "scatter" else DynamicVFE)(**kw).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for layer in m.vfe_layers:
            lin, bn = layer.linear, layer.norm
            n = bn.num_features
            bn.running_mean.copy_(torch.randn(n, generator=g) * 0.5)
            bn.running_var.copy_(torch.rand(n, generator=g) * 1.5 + 0.5)
            bn.weight.copy_(torch.randn(n, generator=g))
            bn.bias.copy_(torch.randn(n, generator=g) * 0.3)
            lin.weight[:2] *= 1e-4  # channel 0: always 0 after the ReLU, channel 1: always active
            bn.running_mean[:2] = 0.0
            bn.weight[:2] = 1.0
            bn.bias[0], bn.bias[1] = -1.0, 1.0
    return m


def _weights64(m):
    return {k: v.detach().double().cpu() for k, v in m.state_dict().items()}


def _reference(cls, m, pts, co, mode):
    """(features, coordinates, inverse or None, point -> output row) in float64 from the oracle"""
    w = _weights64(m)
    nl = len(m.vfe_layers)
    if cls == "scatter":
        vf, vc, inv = O.dynamic_scatter_vfe_forward(pts.double(), co, w, VS, RNG, nl, m._with_cluster_center, m._with_voxel_center,
                                                    mode=mode, eps=EPS, rel_dist_scaler=m.rel_dist_scaler)
        return vf, vc, inv, inv
    vf, vc = O.dynamic_vfe_forward(pts.double(), co.int(), w, VS, RNG, nl, m._with_cluster_center, m._with_voxel_center, mode=mode,
                                   eps=EPS)
    key = lambda c: ((c[:, 0] * GRID_ZYX[0] + c[:, 1]) * GRID_ZYX[1] + c[:, 2]) * GRID_ZYX[2] + c[:, 3]  # noqa: E731
    vk, pk = key(vc.long()), key(co.long())
    row = torch.searchsorted(vk, pk).clamp(max=max(vk.numel() - 1, 0))
    found = (co[:, 1:] >= 0).all(1) & (vk.numel() > 0)
    if vk.numel():
        found &= vk[row] == pk
    return vf, vc, None, torch.where(found, row, torch.full_like(row, -1))


def _bound(m, pts, co, row, M):
    """per output row: the inf-norm of the float64 magnitude propagated through decoration, layers and pooling"""
    keep = row >= 0
    r, x, c = row[keep], pts[keep].double(), co[keep].double()
    mags = [x.abs()]
    if m._with_cluster_center:
        cnt = torch.bincount(r, minlength=M).clamp(min=1).double()[:, None]
        mean = torch.zeros((M, 3), dtype=torch.float64).index_add(0, r, x[:, :3]) / cnt
        mags.append((x[:, :3].abs() + mean[r].abs()) / m.rel_dist_scaler)
    if m._with_voxel_center:
        vs = torch.tensor(VS, dtype=torch.float64)
        off = vs / 2 + torch.tensor(RNG[:3], dtype=torch.float64)
        mags.append(x[:, :3].abs() + (c[:, [3, 2, 1]] * vs).abs() + off.abs())
    h = torch.cat(mags, 1)
    w = _weights64(m)
    for i in range(len(m.vfe_layers)):
        p = f"vfe_layers.{i}."
        s = w[p + "norm.weight"] / torch.sqrt(w[p + "norm.running_var"] + EPS)
        pt = h @ w[p + "linear.weight"].abs().T * s.abs() + w[p + "norm.bias"].abs() + (w[p + "norm.running_mean"] * s).abs()
        pooled = torch.zeros((M, pt.shape[1]), dtype=torch.float64).scatter_reduce(0, r[:, None].expand_as(pt), pt, "amax",
                                                                                   include_self=False)
        h = torch.cat([pt, pooled[r]], 1)
    return pooled.amax(1)


def _launch(cls, m, pts, co, batch):
    """one call of the C entry point with the module's own cfg, into outputs prefilled with sentinels"""
    from sst_b200 import _lib as L
    dev = pts.device
    P, Cout = pts.shape[0], m.feat_channels[-1]
    cfg = m._cfg(batch)
    hi = co[:, 1:].amax(0).tolist()
    for i in range(3):  # like DynamicScatterVFE.forward (no-op for coordinates inside the canvas)
        cfg.grid_zyx[i] = max(cfg.grid_zyx[i], int(hi[i]) + 1)
    vf = torch.full((P, Cout), SENTINEL, device=dev)
    vc = torch.full((P, 4), -7, dtype=torch.int64 if cls == "scatter" else torch.int32, device=dev)
    inv = torch.full((P,), -7, dtype=torch.int64, device=dev)
    num_dev = torch.empty((1,), dtype=torch.int32, device=dev)
    num = C.c_int32(-1)
    c = L.ctx(dev)
    if cls == "scatter":
        rc = L.lib().sstb200_dynamic_scatter_vfe_forward(c, C.byref(cfg), pts.data_ptr(), co.data_ptr(), P, vf.data_ptr(),
                                                         vc.data_ptr(), inv.data_ptr(), num_dev.data_ptr(), C.byref(num))
    else:
        rc = L.lib().sstb200_dynamic_vfe_forward(c, C.byref(cfg), pts.data_ptr(), co.data_ptr(), P, vf.data_ptr(), vc.data_ptr(),
                                                 num_dev.data_ptr(), C.byref(num))
    L.check(c, rc)
    torch.cuda.synchronize()
    assert int(num_dev.item()) == num.value
    return vf, vc, inv, num.value


def _poisoned_twin(m):
    """the same module with every BatchNorm shift raised by POISON: a call with it leaves large positive values in the
    layer-0 voxel features and the other scratch at the arena offsets the next call of the same size uses"""
    t = copy.deepcopy(m)
    with torch.no_grad():
        for layer in t.vfe_layers:
            layer.norm.bias += POISON
    return t


def _check(cls, m, pts, co, mode, precision, cuda, poison=True):
    """run on a dirty workspace and a sentinel-filled output, compare with float64; returns the device outputs"""
    m = m.to(cuda)
    m.precision = precision
    batch = int(co[:, 0].max()) + 1 if cls == "scatter" else int(co[-1, 0]) + 1
    pd, cd = pts.to(cuda), (co if cls == "scatter" else co.int()).contiguous().to(cuda)
    if poison:
        tw = _poisoned_twin(m)
        tw.precision = precision
        _launch(cls, tw, pd, cd, batch)
    vf, vc, inv, M = _launch(cls, m, pd, cd, batch)
    ref, rc, rinv, row = _reference(cls, m, pts, co, mode)
    assert M == ref.shape[0]
    assert torch.equal(vc[:M].cpu(), rc.to(vc.dtype))
    if cls == "scatter":
        assert torch.equal(inv.cpu(), rinv)
    assert bool((vf[M:] == SENTINEL).all()) and bool((vc[M:] == -7).all()), "rows beyond the voxel count were written"
    got = vf[:M].cpu().double()
    assert torch.isfinite(got).all()
    if M:
        bound = _bound(m, pts, co, row, M)
        err = (got - ref).abs().amax(1)
        bf16_l1 = precision == "bf16" and mode == "max" and tuple(m.feat_channels) in TILE_L1 and m.in_channels <= 16
        tol = ROW_TOL["bf16" if bf16_l1 else "fp32"]
        bad = torch.nonzero(err > tol * bound).flatten()
        assert bad.numel() == 0, (f"{bad.numel()} of {M} rows beyond {tol:g} x bound; worst row {int(bad[0])}: err "
                                  f"{err[bad[0]].item():.3e} bound {bound[bad[0]].item():.3e}")
        rel = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)
        assert rel < MAX_TOL["bf16" if bf16_l1 else "fp32"], rel
    return vf[:M], vc[:M], inv, M


def _routes():
    out = []
    for c0, c1 in FUSED:
        for mode in ("max", "avg"):
            out.append((c0, c1, mode, "fp32"))
            if mode == "max" and (c0, c1) in TILE_L1:
                out.append((c0, c1, mode, "bf16"))
    return out


CLASSES = ("dynamic", "scatter")


# ----------------------------------------------------------------------------------------------------------------------
# tests
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("c0,c1,mode,precision", _routes())
def test_routes(cuda, cls, c0, c1, mode, precision):
    """every instantiated (C0, C1) x max / avg (x bf16 where it selects the tensor-core layer 1) on the edge layout"""
    pts, co = _cloud(_layout("edges"), 4, 100 + c0 + c1, cls == "dynamic")
    _check(cls, _module(cls, 4, c0, c1, mode, seed=c0 + c1), pts, co, mode, precision, cuda)


@pytest.mark.parametrize("cls", CLASSES)
def test_uninstantiated_pair_raises(cuda, cls):
    from sst_b200._lib import SSTB200Error
    pts, co = _cloud(_layout("total_128"), 4, 3, cls == "dynamic")
    m = _module(cls, 4, 48, 64, "max").to(cuda)
    with pytest.raises(SSTB200Error, match=r"\(48,64\) not instantiated"):
        m(pts.to(cuda), co.to(cuda))
    m = _module(cls, 4, 64, 128, "max").to(cuda)  # the context stays usable
    assert m(pts.to(cuda), co.to(cuda))[0].shape[1] == 128


DECORATIONS = [(4, False, False), (4, True, False), (4, False, True), (4, True, True),
               (10, True, True), (11, True, True),        # D0 = 16 (tile / fused) | 17 (wide)
               (16, False, False), (17, False, False)]


@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("F,cluster,centre", DECORATIONS)
@pytest.mark.parametrize("c0,c1,mode,precision", [(64, 128, "max", "fp32"), (64, 128, "max", "bf16"), (64, 64, "avg", "fp32")])
def test_decoration(cuda, cls, F, cluster, centre, c0, c1, mode, precision):
    """cluster / centre on and off; D0 = 16 against 17 (the wide route) reached with and without decorations"""
    pts, co = _cloud(_layout("edges"), F, 200 + F, cls == "dynamic")
    _check(cls, _module(cls, F, c0, c1, mode, cluster, centre, seed=F), pts, co, mode, precision, cuda)


LAYOUT_CFGS = [(32, 64, "max", "fp32"), (32, 64, "max", "bf16"), (64, 128, "max", "bf16"), (64, 0, "max", "fp32"),
               (32, 32, "max", "fp32"), (128, 128, "avg", "fp32")]


@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("layout", ["edges", "one_point", "big_voxel", "total_1", "total_127", "total_128", "total_129", "persistent"])
@pytest.mark.parametrize("c0,c1,mode,precision", LAYOUT_CFGS)
def test_layouts(cuda, cls, layout, c0, c1, mode, precision):
    """voxel boundaries on and across every row-group and tile edge, one voxel of one point, a voxel over three tiles, tiny valid
    totals and a second pass of the persistent tile loops"""
    pts, co = _cloud(_layout(layout), 4, 300 + c0 + c1, cls == "dynamic")
    _check(cls, _module(cls, 4, c0, c1, mode, seed=7), pts, co, mode, precision, cuda)


BATCH_CFGS = [(4, 64, 128, "max", "bf16"), (4, 32, 64, "max", "fp32"), (4, 64, 64, "avg", "fp32"), (11, 64, 128, "max", "fp32")]


@pytest.mark.parametrize("F,c0,c1,mode,precision", BATCH_CFGS)
def test_batch_dynamic_vfe(cuda, F, c0, c1, mode, precision):
    """DynamicVFE, batch of 4: sample 1 has only out-of-range points, sample 2 one voxel that the drop-first rule removes, sample 3
    out-of-range points beside its voxels (its (-1,-1,-1) row is the one removed, so it keeps all its voxels)"""
    counts = [_random_counts(1, 300, 9), [], [], _random_counts(2, 200, 9)]
    pts, co = _cloud(counts, F, 17, True, invalid={1: 40, 3: 25})
    p2, c2 = _cloud([[], [], [5]], F, 18, False)  # sample 2: exactly one voxel, no out-of-range point
    pts, co = torch.cat([p2, pts]), torch.cat([c2, co])
    m = _module("dynamic", F, c0, c1, mode, seed=3)
    _, vc, _, _ = _check("dynamic", m, pts, co, mode, precision, cuda)
    assert set(vc[:, 0].tolist()) == {0, 3}
    assert (vc[:, 0] == 3).sum() == len(counts[3])


@pytest.mark.parametrize("F,c0,c1,mode,precision", BATCH_CFGS)
def test_batch_dynamic_scatter_vfe(cuda, F, c0, c1, mode, precision):
    """DynamicScatterVFE, batch of 4: sample 1 empty, sample 2 one voxel"""
    pts, co = _cloud([_random_counts(3, 300, 9), [], [4], _random_counts(4, 150, 9)], F, 19, False)
    _, vc, _, _ = _check("scatter", _module("scatter", F, c0, c1, mode, seed=4), pts, co, mode, precision, cuda)
    assert (vc[:, 0] == 2).sum() == 1 and (vc[:, 0] == 1).sum() == 0


@pytest.mark.parametrize("F", [4, 11])
def test_all_points_out_of_range(cuda, F):
    """DynamicVFE with every point out of range: no voxel, empty outputs, nothing written"""
    g = torch.Generator().manual_seed(5)
    pts = torch.randn((300, F), generator=g) * 30
    co = torch.tensor([[0, -1, -1, -1]] * 150 + [[1, -1, -1, -1]] * 150, dtype=torch.int32)
    m = _module("dynamic", F, 64, 128, "max").to(cuda)
    vf, vc = m(pts.to(cuda), co.to(cuda))
    assert vf.shape == (0, 128) and vc.shape == (0, 4)
    vf, vc, _, M = _launch("dynamic", m, pts.to(cuda), co.to(cuda), 2)
    assert M == 0 and bool((vf == SENTINEL).all()) and bool((vc == -7).all())


@pytest.mark.parametrize("cls", CLASSES)
@pytest.mark.parametrize("c0,c1,mode,precision", [(64, 128, "max", "fp32"), (64, 128, "max", "bf16"), (32, 64, "max", "fp32"),
                                                  (64, 64, "avg", "fp32"), (128, 0, "max", "fp32")])
def test_repeatable(cuda, cls, c0, c1, mode, precision):
    """max pooling: two calls give bit-identical features (per-point values do not depend on the CSR fill order, the max is exact
    and wgmma rows are independent); mean: the same within the bound (the CSR fill order is atomic)"""
    pts, co = _cloud(_layout("edges"), 4, 400, cls == "dynamic")
    m = _module(cls, 4, c0, c1, mode, seed=9)
    a = _check(cls, m, pts, co, mode, precision, cuda)[0].clone()
    b = _check(cls, m, pts, co, mode, precision, cuda, poison=False)[0]
    if mode == "max":
        assert torch.equal(a, b)
