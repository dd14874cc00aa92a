"""GPU: the SST BEV canvas (csrc/bev.cu: sstb200_recover_bev and _backward) and FSD's voxel-to-point neck (csrc/neck.cu:
sstb200_voxel2point and _backward) against oracle/sst_oracle at every tile, scan and alignment edge, through the C ABI.

recover_bev transposes 128-cell x 32-channel tiles through shared memory and writes each canvas row with float4 streaming stores
when every row starts 16-byte aligned (nx % 4 == 0 and an aligned canvas), with scalar stores otherwise; its backward reads the
gradient the same way.  The cases run nx on both sides of the float4 split and of the 128-cell block, C on both sides of the
32-channel pass up to the 1024 limit, empty, one-voxel-per-block and full canvases, duplicated cells, out-of-canvas coordinates,
and canvases and gradients at 4-, 8- and 12-byte offsets.  The neck builds a keep mask (one warp per point), compacts it with the
look-back scan (SCAN_TILE points per tile, read from common.cuh) and sums the kept points' gradients per voxel in fp64; the cases
put N and K on both sides of the scan tiles, keep nothing and everything, pad with 0.0 (-0.0 rows count as padded, as == gives)
and with NaN (never padded), and reference one voxel from 1e5 points.

Every comparison is exact.  The forwards are copies plus the reference's fp32 expression, so the canvas is compared bit for bit.
The backward gradients are compared with float64 autograd: recover_bev's is a copy, and the neck's inputs are small integers times
2^-6, so the fp64 sum is exact and its fp32 rounding unique.  Every output is prefilled with a sentinel (NaN for the canvas and
grad_voxel) and has guard space past its end that must keep it, and every call runs after a larger "poison twin" on the same
context, so the arena it carves is dirty.
"""
import ctypes as C
import os
import re

import pytest
import torch

from oracle import sst_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 64        # floats past the canvas
GUARD_ROWS = 4    # rows past grad_feat, out and grad_voxel
SENTINEL = -1234.5
NAN = float("nan")


def _lib():
    from sst_b200 import _lib as L
    from sst_b200 import neck_modules, sst_modules  # noqa: F401  (bind the four entry points)
    return L


def _bits(t):
    return t.contiguous().view(torch.int32)


def scan_tile():
    src = open(os.path.join(ROOT, "sst_b200", "csrc", "common.cuh")).read()
    items = int(re.search(r"#define SCAN_ITEMS (\d+)", src).group(1))
    threads = int(re.search(r"#define SCAN_THREADS (\d+)", src).group(1))
    assert re.search(r"#define SCAN_TILE \(SCAN_ITEMS \* SCAN_THREADS\)", src)
    assert "launch_exclusive_scan(c->stream, LoadU32{keep}" in open(os.path.join(ROOT, "sst_b200", "csrc", "neck.cu")).read()
    return items * threads


# ---- recover_bev ------------------------------------------------------------------------------------------------------------------
def _cells(B, ny, nx, mode, seed):
    """coors [M, 4] (b, 0, y, x): none, one voxel in each 128-cell block of each (b, y) row, or every cell (random row order)"""
    g = torch.Generator().manual_seed(seed)
    if mode == "empty":
        return torch.zeros((0, 4), dtype=torch.long)
    if mode == "block":
        rows = []
        for b in range(B):
            for y in range(ny):
                for x0 in range(0, nx, 128):
                    x = x0 + int(torch.randint(0, min(128, nx - x0), (1,), generator=g))
                    rows.append((b, 0, y, x))
        co = torch.tensor(rows, dtype=torch.long)
    else:
        b, y, x = torch.meshgrid(torch.arange(B), torch.arange(ny), torch.arange(nx), indexing="ij")
        co = torch.stack([b.flatten(), torch.zeros(B * ny * nx, dtype=torch.long), y.flatten(), x.flatten()], 1)
    return co[torch.randperm(co.shape[0], generator=g)].contiguous()


def bev_forward(c, dev, feat, coors, B, ny, nx, offset=0):
    """canvas at `offset` floats into a NaN-filled buffer with GUARD floats past its end; returns the canvas (CPU)"""
    L = _lib()
    M, C_ = feat.shape
    total = B * C_ * ny * nx
    buf = torch.full((offset + total + GUARD,), NAN, device=dev)
    f, co = feat.contiguous().to(dev), coors.contiguous().to(dev)
    L.check(c, L.lib().sstb200_recover_bev(c, L.ptr(f) if M else None, L.ptr(co) if M else None, M, C_, B, ny, nx,
                                           buf.data_ptr() + 4 * offset))
    buf = buf.cpu()
    assert torch.isnan(buf[:offset]).all() and torch.isnan(buf[offset + total:]).all(), "a float outside the canvas was written"
    canvas = buf[offset:offset + total].view(B, C_, ny, nx)
    assert not torch.isnan(canvas).any(), "a canvas element was not written"
    return canvas


def bev_backward(c, dev, grad, coors, C_, offset=0):
    """grad_canvas at `offset` floats into a larger buffer; grad_feat prefilled with SENTINEL plus GUARD_ROWS rows"""
    L = _lib()
    B, _, ny, nx = grad.shape
    M = coors.shape[0]
    flat = torch.empty((offset + grad.numel() + GUARD,), device=dev).fill_(SENTINEL)
    flat[offset:offset + grad.numel()] = grad.flatten().to(dev)
    out = torch.full((M + GUARD_ROWS, C_), SENTINEL, device=dev)
    co = coors.contiguous().to(dev)
    L.check(c, L.lib().sstb200_recover_bev_backward(c, flat.data_ptr() + 4 * offset, L.ptr(co) if M else None, M, C_, B, ny, nx,
                                                    out.data_ptr()))
    out = out.cpu()
    assert (out[M:] == SENTINEL).all(), "a guard row past M was written"
    return out[:M]


def _bev_poison(c, dev, C_, B, ny, nx):
    """a larger forward and backward (more channels, cells and voxels) on the same context"""
    Cp, Bp, nyp, nxp = min(C_ + 9, 1024), B + 1, ny + 2, nx + 37
    g = torch.Generator().manual_seed(C_ + nx)
    co = _cells(Bp, nyp, nxp, "block", C_)
    co = torch.cat([co, co[: co.shape[0] // 2]])
    feat = torch.randn(co.shape[0], Cp, generator=g) * 1e4
    bev_forward(c, dev, feat, co, Bp, nyp, nxp)
    bev_backward(c, dev, torch.randn(Bp, Cp, nyp, nxp, generator=g) * 1e4, co, Cp)


def _bev_ref_grad(feat, coors, B, ny, nx, probe):
    xo = feat.double().requires_grad_(True)
    (O.recover_bev(xo, coors, B, (ny, nx)) * probe.double()).sum().backward()
    return xo.grad.float()


NX = [1, 3, 4, 127, 128, 129, 255, 256, 257, 468]
CH = [1, 31, 32, 33, 64, 65, 1024]
LAYOUT = [("empty", 2, 1), ("block", 3, 2), ("full", 4, 1)]


@pytest.mark.parametrize("nx", NX)
@pytest.mark.parametrize("C_", CH)
def test_recover_bev_shapes(cuda, nx, C_):
    """forward bit-exact against the oracle (every canvas element written, zeros included, no guard float touched) and backward
    bit-exact against float64 autograd, for an empty canvas, one voxel per 128-cell block and every cell occupied"""
    L = _lib()
    c = L.ctx(cuda)
    for mode, B, ny in LAYOUT:
        coors = _cells(B, ny, nx, mode, seed=nx * 7 + C_)
        g = torch.Generator().manual_seed(nx + C_)
        feat = torch.randn(coors.shape[0], C_, generator=g)
        ref = O.recover_bev(feat, coors, B, (ny, nx))
        _bev_poison(c, cuda, C_, B, ny, nx)
        got = bev_forward(c, cuda, feat, coors, B, ny, nx)
        assert torch.equal(_bits(got), _bits(ref)), f"{mode}: canvas differs"
        if mode == "empty":
            continue
        probe = torch.randn(B, C_, ny, nx, generator=g)
        _bev_poison(c, cuda, C_, B, ny, nx)
        gf = bev_backward(c, cuda, probe, coors, C_)
        assert torch.equal(_bits(gf), _bits(_bev_ref_grad(feat, coors, B, ny, nx, probe))), f"{mode}: grad_feat differs"
    # M = 0 backward writes nothing
    out = bev_backward(c, cuda, torch.randn(1, C_, 1, nx), torch.zeros((0, 4), dtype=torch.long), C_)
    assert out.shape[0] == 0


@pytest.mark.parametrize("nx", [4, 129, 256])
def test_recover_bev_duplicates_and_out_of_canvas(cuda, nx):
    """duplicated cells hold one of their rows, and each of those rows receives the cell's gradient; a coordinate outside the canvas
    in b, y or x on either side is refused by the forward and gets a zero gradient row in the backward"""
    L = _lib()
    c = L.ctx(cuda)
    B, ny, C_ = 2, 3, 40
    co = _cells(B, ny, nx, "block", seed=nx)
    co = torch.cat([co, _cells(B, ny, nx, "full", seed=nx + 1)[: 2 * nx]])
    dup = torch.cat([co, co[: co.shape[0] // 3]])
    dup = dup[torch.randperm(dup.shape[0], generator=torch.Generator().manual_seed(nx))]
    g = torch.Generator().manual_seed(3 * nx)
    feat = torch.randn(dup.shape[0], C_, generator=g)
    _bev_poison(c, cuda, C_, B, ny, nx)
    got = bev_forward(c, cuda, feat, dup, B, ny, nx)
    key = (dup[:, 0] * ny + dup[:, 2]) * nx + dup[:, 3]
    uk, inv = torch.unique(key, return_inverse=True)
    flat = got.permute(0, 2, 3, 1).reshape(B * ny * nx, C_)
    held = flat[key]
    for k in range(uk.numel()):  # the cell holds exactly one of the rows that map to it
        rows = feat[inv == k]
        assert (rows == held[inv == k][0]).all(1).any()
    empty = torch.ones(B * ny * nx, dtype=torch.bool)
    empty[uk] = False
    assert (flat[empty] == 0).all() and not torch.signbit(flat[empty]).any()
    probe = torch.randn(B, C_, ny, nx, generator=g)
    _bev_poison(c, cuda, C_, B, ny, nx)
    gf = bev_backward(c, cuda, probe, dup, C_)
    assert torch.equal(_bits(gf), _bits(_bev_ref_grad(feat, dup, B, ny, nx, probe)))
    # out-of-canvas coordinates
    for col, bad in ((0, -1), (0, B), (2, -1), (2, ny), (3, -1), (3, nx)):
        co_bad = dup.clone()
        pos = [0, dup.shape[0] // 2, dup.shape[0] - 1]
        co_bad[pos, col] = bad
        _bev_poison(c, cuda, C_, B, ny, nx)
        with pytest.raises(L.SSTB200Error):
            bev_forward(c, cuda, feat, co_bad, B, ny, nx)
        _bev_poison(c, cuda, C_, B, ny, nx)
        gf = bev_backward(c, cuda, probe, co_bad, C_)
        ok = torch.ones(dup.shape[0], dtype=torch.bool)
        ok[pos] = False
        ref = torch.zeros_like(gf)
        ref[ok] = _bev_ref_grad(feat[ok], co_bad[ok], B, ny, nx, probe)
        assert torch.equal(_bits(gf), _bits(ref)), (col, bad)
    with pytest.raises(L.SSTB200Error):  # 1025 channels
        bev_forward(c, cuda, torch.zeros((1, 1025)), torch.zeros((1, 4), dtype=torch.long), 1, 1, nx)


@pytest.mark.parametrize("nx", [4, 128, 256, 468, 257])
def test_recover_bev_misaligned(cuda, nx):
    """the canvas and grad_canvas 4, 8 and 12 bytes past a 16-byte boundary: the same bits as the aligned call (the float4 rows
    need 16-byte alignment, so these take the scalar path)"""
    L = _lib()
    c = L.ctx(cuda)
    B, ny, C_ = 2, 3, 37
    co = _cells(B, ny, nx, "block", seed=nx)
    co = torch.cat([co, _cells(B, ny, nx, "full", seed=nx + 5)[: nx + 3]])
    co = torch.unique(co, dim=0)
    g = torch.Generator().manual_seed(nx)
    feat = torch.randn(co.shape[0], C_, generator=g)
    probe = torch.randn(B, C_, ny, nx, generator=g)
    ref = O.recover_bev(feat, co, B, (ny, nx))
    ref_g = _bev_ref_grad(feat, co, B, ny, nx, probe)
    for off in (0, 1, 2, 3):
        _bev_poison(c, cuda, C_, B, ny, nx)
        assert torch.equal(_bits(bev_forward(c, cuda, feat, co, B, ny, nx, offset=off)), _bits(ref)), off
        _bev_poison(c, cuda, C_, B, ny, nx)
        assert torch.equal(_bits(bev_backward(c, cuda, probe, co, C_, offset=off)), _bits(ref_g)), off


def test_recover_bev_offset_gradient_through_autograd(cuda):
    """a contiguous canvas gradient that starts 4 bytes into its storage reaches sstb200_recover_bev_backward unchanged through
    _RecoverBevFunction: the row gradients equal float64 autograd"""
    from sst_b200.sst_modules import SSTv2
    B, C_, ny, nx = 2, 48, 5, 256
    co = _cells(B, ny, nx, "block", seed=1)
    co = torch.unique(torch.cat([co, _cells(B, ny, nx, "full", seed=2)[:300]]), dim=0)
    g = torch.Generator().manual_seed(4)
    feat = torch.randn(co.shape[0], C_, generator=g)
    probe = torch.randn(B, C_, ny, nx, generator=g)
    m = SSTv2(d_model=[C_], nhead=[1], num_blocks=0, dim_feedforward=[C_], output_shape=[ny, nx], num_attached_conv=0, to_bev=True)
    storage = torch.empty(probe.numel() + 1, device=cuda)
    gview = storage[1:].view(B, C_, ny, nx)
    gview.copy_(probe.to(cuda))
    assert gview.is_contiguous() and gview.data_ptr() % 16 == 4
    x = feat.to(cuda).requires_grad_(True)
    _bev_poison(_lib().ctx(cuda), cuda, C_, B, ny, nx)
    m.recover_bev(x, co.to(cuda), B).backward(gview)
    assert torch.equal(_bits(x.grad.cpu()), _bits(_bev_ref_grad(feat, co, B, ny, nx, probe)))


# ---- Voxel2PointScatterNeck -------------------------------------------------------------------------------------------------------
VS = (0.32, 0.32, 6.0)
RNG = [-74.88, -74.88, -2.0, 74.88, 74.88, 4.0]
GRID = (468, 468, 1)


def _neck_inputs(N, M, C_, seed, padding=-1.0, pad_every=7):
    """points inside their voxels (coordinates up to the grid's last cell), voxel rows with every pad_every-th one padded"""
    g = torch.Generator().manual_seed(seed)
    co = torch.stack([torch.randint(0, 2, (N,), generator=g), torch.randint(0, GRID[2], (N,), generator=g),
                      torch.randint(0, GRID[1], (N,), generator=g), torch.randint(0, GRID[0], (N,), generator=g)], 1)
    co[: N // 4, 1:] = torch.tensor([GRID[2] - 1, GRID[1] - 1, GRID[0] - 1])
    vs, mn = torch.tensor(VS), torch.tensor(RNG[:3])
    pts = ((co[:, [3, 2, 1]].float() + torch.rand((N, 3), generator=g)) * vs + mn).float()
    pts = torch.cat([pts, torch.rand((N, 2), generator=g)], 1)
    vf = torch.randn(M, C_, generator=g)
    if pad_every:
        vf[::pad_every] = padding
    inds = torch.randint(0, M, (N,), generator=g)
    return pts, co, vf, inds


def v2p_forward(c, dev, pts, co, vf, inds, padding=-1.0, with_xyz=True, normalize=False):
    """out prefilled with SENTINEL plus GUARD_ROWS rows, mask with 7s; returns (out [N + GUARD_ROWS], mask [N], K)"""
    L = _lib()
    N, (M, C_) = pts.shape[0], vf.shape
    Co = C_ + (3 if with_xyz else 0)
    out = torch.full((N + GUARD_ROWS, Co), SENTINEL, device=dev)
    mask = torch.full((N + GUARD_ROWS,), 7, dtype=torch.uint8, device=dev)
    num_dev = torch.full((1,), -1, dtype=torch.int32, device=dev)
    num = C.c_int32(-1)
    p, cd, v, i = (t.contiguous().to(dev) for t in (pts, co, vf, inds))
    L.check(c, L.lib().sstb200_voxel2point(c, p.data_ptr(), pts.shape[1], cd.data_ptr(), v.data_ptr(), M, C_, i.data_ptr(), N, float(padding),
                                           L.arr(C.c_float, list(VS)), L.arr(C.c_float, RNG[:3]), int(with_xyz), int(normalize),
                                           out.data_ptr(), mask.data_ptr(), num_dev.data_ptr(), C.byref(num)))
    out, mask = out.cpu(), mask.cpu()
    assert (mask[N:] == 7).all() and int(num_dev.item()) == num.value
    return out, mask[:N], num.value


def v2p_backward(c, dev, gout, mask, inds, M, C_, with_xyz):
    """grad_voxel prefilled with NaN plus GUARD_ROWS rows"""
    L = _lib()
    K, N = gout.shape[0], inds.shape[0]
    out = torch.full((M + GUARD_ROWS, C_), NAN, device=dev)
    g, m, i = gout.contiguous().to(dev), mask.contiguous().to(dev), inds.contiguous().to(dev)
    L.check(c, L.lib().sstb200_voxel2point_backward(c, g.data_ptr(), m.data_ptr(), i.data_ptr(), N, K, M, C_, int(with_xyz), out.data_ptr()))
    out = out.cpu()
    assert torch.isnan(out[M:]).all(), "a guard row past M was written"
    return out[:M]


def _neck_poison(c, dev, N, M, C_):
    pts, co, vf, inds = _neck_inputs(N + 517, M + 33, C_ + 5, seed=N + C_, pad_every=3)
    vf *= 1e4
    out, mask, K = v2p_forward(c, dev, pts, co, vf, inds)
    v2p_backward(c, dev, torch.randn(K, C_ + 8) * 1e4, mask.bool().to(torch.uint8), inds, M + 33, C_ + 5, True)


def _dyadic(shape, seed):
    return torch.randint(-64, 65, shape, generator=torch.Generator().manual_seed(seed)).float() * 2.0 ** -6


def neck_case(dev, pts, co, vf, inds, padding=-1.0, with_xyz=True, normalize=False, seed=0):
    """forward bit-exact against the oracle (rows K..N-1 keep the sentinel), backward against float64 autograd; returns (mask, K)"""
    L = _lib()
    c = L.ctx(dev)
    N, (M, C_) = pts.shape[0], vf.shape
    ref, ref_mask = O.voxel2point_neck(pts, co, vf, inds, VS, RNG, with_xyz, normalize, padding)
    _neck_poison(c, dev, N, M, C_)
    out, mask, K = v2p_forward(c, dev, pts, co, vf, inds, padding, with_xyz, normalize)
    assert K == int(ref_mask.sum()) and torch.equal(mask.bool(), ref_mask)
    assert torch.equal(_bits(out[:K]), _bits(ref)), "neck rows differ"
    assert (out[K:] == SENTINEL).all(), "a row past K was written"
    gout = _dyadic((K, out.shape[1]), seed)
    xo = vf.double().requires_grad_(True)
    o, _ = O.voxel2point_neck(pts.double(), co, xo, inds, VS, RNG, with_xyz, normalize, padding)
    (o * gout.double()).sum().backward()
    _neck_poison(c, dev, N, M, C_)
    got = v2p_backward(c, dev, gout, mask, inds, M, C_, with_xyz)
    assert torch.equal(got, xo.grad.float()), "grad_voxel differs"
    cnt = torch.bincount(inds[ref_mask], minlength=M)
    assert (got[cnt == 0] == 0).all()
    return ref_mask, K


@pytest.mark.parametrize("tiles", [(0, 1), (1, -1), (1, 0), (1, 1), (2, -1), (2, 0), (2, 1), (3, 5)])
def test_voxel2point_scan_tiles(cuda, tiles):
    """N = a * SCAN_TILE + b: the look-back scan's tile edges, with about 1 in 7 points dropped (K on both sides too), and with
    everything kept (K = N)"""
    T = scan_tile()
    N = tiles[0] * T + tiles[1]
    M = max(N // 3, 1)
    pts, co, vf, inds = _neck_inputs(N, M, 33, seed=N)
    mask, K = neck_case(cuda, pts, co, vf, inds, seed=N)
    assert 0 < K < N or N == 1
    pts, co, vf, inds = _neck_inputs(N, M, 33, seed=N + 1, pad_every=0)
    _, K = neck_case(cuda, pts, co, vf, inds, seed=N + 1)
    assert K == N


@pytest.mark.parametrize("C_", [1, 31, 32, 33, 300])
@pytest.mark.parametrize("with_xyz,normalize", [(True, False), (True, True), (False, False)])
def test_voxel2point_channels(cuda, C_, with_xyz, normalize):
    T = scan_tile()
    pts, co, vf, inds = _neck_inputs(T + 1, 700, C_, seed=C_)
    neck_case(cuda, pts, co, vf, inds, with_xyz=with_xyz, normalize=normalize, seed=C_)


def test_voxel2point_padding_values(cuda):
    """padding 0.0: rows of -0.0 and of +0.0 are padded (== compares them equal), a row with one non-zero is kept; padding NaN:
    nothing is padded, NaN rows included; everything padded gives K = 0 and zero gradients"""
    N, M, C_ = 3000, 400, 33
    pts, co, vf, inds = _neck_inputs(N, M, C_, seed=5, pad_every=0)
    vf[::5] = -0.0
    vf[1::5] = 0.0
    vf[2::10] = 0.0
    vf[2::10, 7] = 1.0
    mask, _ = neck_case(cuda, pts, co, vf, inds, padding=0.0, seed=5)
    assert not mask[(inds % 5 == 0) | (inds % 5 == 1)].any() and mask[inds % 10 == 2].all()
    vf2 = vf.clone()
    vf2[3::9] = NAN
    _, K = neck_case(cuda, pts, co, vf2, inds, padding=NAN, with_xyz=False, seed=6)
    assert K == N
    vf3 = torch.full((M, C_), -1.0)
    _, K = neck_case(cuda, pts, co, vf3, inds, seed=7)
    assert K == 0


def test_voxel2point_backward_hot_voxel(cuda):
    """one voxel referenced by 1e5 points, many voxels by none, padded voxels: exact sums, exact zeros"""
    N, M, C_ = 100000, 5000, 64
    pts, co, vf, inds = _neck_inputs(N + 20000, M, C_, seed=9)
    inds[:N] = 1
    _, K = neck_case(cuda, pts, co, vf, inds, seed=9)
    assert K >= N


def test_voxel2point_refuses_out_of_range_index(cuda):
    """an index outside [0, M) in the first or the last position is refused"""
    L = _lib()
    c = L.ctx(cuda)
    pts, co, vf, inds = _neck_inputs(3000, 400, 16, seed=11)
    for pos in (0, -1):
        for bad in (-1, 400):
            i = inds.clone()
            i[pos] = bad
            _neck_poison(c, cuda, 3000, 400, 16)
            with pytest.raises(L.SSTB200Error):
                v2p_forward(c, cuda, pts, co, vf, i)
