"""GPU: the sparse convolution kernels (csrc/spconv.cu) against float64 at every tile edge and operand scale.

Kernels tile rows by 64 (fp32 FFMA), 128 (wgmma, two 64-row warpgroups) and 1024 (weight gradient), channels by 16 / 64 / 128; the
cases below sit on both sides of each of those edges, on every kernel volume the layer classes can produce, on degenerate tables
(dense grid, single voxel, empty samples, a tile without any pair) and on a key space beyond 2^31 cells.

Reference: oracle.spconv_oracle (tables bit-exact, features in float64) and the float64 restatements `_ref_conv` / `_ref_dw` /
`_ref_dx` below, written from the neighbour table alone.

Error metric: besides the max-norm of the older tests every comparison asserts a PER-ROW bound
    |out[o] - ref[o]|_inf  <=  tol * |(sum_k |x[nbr[o,k]]| @ |W[k]|) * |scale| + |shift| + |residual[o]||_inf
(the float64 product of absolute values: what a rounding error of the row can be relative to), so a wrong small row cannot hide
behind a large one.  Per-row tolerances: fp32 1e-5, fp32_tc 1e-5, bf16 (IEEE fp16 operands) 5e-3 - at ANY power-of-two scale of
features, weights or gradients (test_scale_*): the tensor-core paths carry exponents beside their fp16 operands."""
import functools

import pytest
import torch

from oracle import spconv_oracle as SO

pytestmark = pytest.mark.gpu

PRECS = ("fp32", "bf16", "fp32_tc")
ROW_TOL = {"fp32": 1e-5, "bf16": 5e-3, "fp32_tc": 1e-5}
MAX_TOL = {"fp32": 1e-4, "bf16": 5e-3, "fp32_tc": 1e-4}
SHAPE, BATCH = [10, 40, 40], 2
K3, S1, P1 = [3, 3, 3], [1, 1, 1], [1, 1, 1]
SENTINEL = -12345.0


# ----------------------------------------------------------------------------------------------------------------------
# data, float64 restatements, launch with guard rows
# ----------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _cloud():
    """one clustered sparse tensor, rows in random order (a tile's neighbours live in other tiles); 320 channels to slice from"""
    feats, coors = SO.synth_sparse(77, BATCH, SHAPE, 1700, 320)
    assert coors.shape[0] >= 3000
    return feats, coors


@functools.lru_cache(maxsize=None)
def _subm_table(n):
    """SubM 3x3x3 table of the first n rows of the cloud (oracle)"""
    coors = _cloud()[1][:n]
    return SO.neighbour_table(coors, coors, BATCH, SHAPE, K3, S1, P1)


def _weights(seed, kv, cin, cout):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn((kv, cin, cout), generator=g) / (kv * cin) ** 0.5 * 2
    return w, torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.3, g


def _ref_conv(x, nbr, w, scale=None, shift=None, res=None, relu=False):
    """(out, bound) in float64: the convolution of sstb200_spconv_forward and the per-row inf-norm of its absolute-value product"""
    x, w = x.double(), w.double()
    acc = torch.zeros((nbr.shape[0], w.shape[2]), dtype=torch.float64)
    mag = torch.zeros_like(acc)
    for k in range(nbr.shape[1]):
        idx = nbr[:, k].long()
        m = idx >= 0
        acc[m] += x[idx[m]] @ w[k]
        mag[m] += x[idx[m]].abs() @ w[k].abs()
    if scale is not None:
        acc, mag = acc * scale.double(), mag * scale.double().abs()
    if shift is not None:
        acc, mag = acc + shift.double(), mag + shift.double().abs()
    if res is not None:
        acc, mag = acc + res.double(), mag + res.double().abs()
    return (acc.clamp_min(0) if relu else acc), mag.amax(1)


def _ref_dw(x, nbr, dy):
    """(dW, bound) float64: dW[k] = X[nbr[:, k]]^T dY over the rows that have a neighbour at k; bound = the same of absolute values"""
    x, dy = x.double(), dy.double()
    dw = torch.zeros((nbr.shape[1], x.shape[1], dy.shape[1]), dtype=torch.float64)
    mag = torch.zeros_like(dw)
    for k in range(nbr.shape[1]):
        idx = nbr[:, k].long()
        m = idx >= 0
        dw[k] = x[idx[m]].T @ dy[m]
        mag[k] = x[idx[m]].abs().T @ dy[m].abs()
    return dw, mag


def _ref_dx(dy, nbr, w, n_in):
    """(dX, bound) float64: dX = scatter of dY W[k]^T along the table; bound per input row"""
    dy, w = dy.double(), w.double()
    dx = torch.zeros((n_in, w.shape[1]), dtype=torch.float64)
    mag = torch.zeros_like(dx)
    for k in range(nbr.shape[1]):
        idx = nbr[:, k].long()
        m = idx >= 0
        dx.index_add_(0, idx[m], dy[m] @ w[k].T)
        mag.index_add_(0, idx[m], dy[m].abs() @ w[k].abs().T)
    return dx, mag.amax(1)


def _transpose_table(nbr, n_in):
    inv = torch.full((n_in, nbr.shape[1]), -1, dtype=torch.int32)
    o, k = torch.nonzero(nbr >= 0, as_tuple=True)
    inv[nbr[o, k].long(), k] = o.int()
    return inv


def _check(out, ref, bound, prec, what="", row_tol=None):
    """per-row condition-aware bound + the max-norm of the older tests"""
    out, tol = out.detach().double().cpu(), (row_tol or ROW_TOL[prec])
    assert out.shape == ref.shape and bool(torch.isfinite(out).all()), what
    err = (out - ref).abs()
    if err.dim() == 2:
        err = err.amax(1)
    worst = int(torch.argmax(err - tol * bound))
    assert bool((err <= tol * bound).all()), (f"{what} {prec}: row {worst} off by {float(err[worst]):.3e}, allowed {tol:g} x "
                                             f"{float(bound[worst]):.3e} (ratio {float(err[worst] / bound[worst].clamp_min(1e-300)):.2e})")
    assert float(err.max()) <= MAX_TOL[prec] * float(ref.abs().max()) + 1e-300, f"{what} {prec}: max-norm"


def _launch(cuda, x, nbr, w, prec, scale=None, shift=None, res=None, relu=False, guard=3):
    """sstb200_spconv_forward through ctypes into the interior of a sentinel-filled buffer; asserts the guard rows are untouched"""
    from sst_b200 import _lib as L, spconv_modules as SP
    dev = lambda t: None if t is None else t.float().contiguous().to(cuda)
    x, w, scale, shift, res, nbr = dev(x), dev(w), dev(scale), dev(shift), dev(res), nbr.to(cuda).contiguous()
    kv, cin, cout = w.shape
    n = nbr.shape[0]
    buf = torch.full((n + 2 * guard, cout), SENTINEL, dtype=torch.float32, device=cuda)
    out = buf[guard:guard + n]
    h16, un = SP._pack_h16(w, prec) if prec != "fp32" else (None, None)
    c = L.ctx(cuda)
    L.check(c, L.lib().sstb200_spconv_forward(c, x.data_ptr(), x.shape[0], cin, nbr.data_ptr(), n, kv, w.data_ptr(), L.ptr(h16), L.ptr(un), cout,
                                              L.ptr(scale), L.ptr(shift), L.ptr(res), int(relu), SP.PREC[prec], out.data_ptr()))
    assert bool((buf[:guard] == SENTINEL).all()) and bool((buf[guard + n:] == SENTINEL).all()), "rows outside [0, n_out) written"
    return out.clone()


# ----------------------------------------------------------------------------------------------------------------------
# a. row-tiling edges, forward
# ----------------------------------------------------------------------------------------------------------------------
ROWS = (1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 1023, 1024, 1025)


@pytest.mark.parametrize("epilogue", [False, True], ids=["plain", "epilogue"])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("cout", [64, 128])
@pytest.mark.parametrize("n", ROWS)
def test_row_edges(cuda, n, cout, prec, epilogue):
    from sst_b200 import spconv_modules as SP
    feats, coors = _cloud()
    x, c, nbr_ref = feats[:n, :64], coors[:n], _subm_table(n)
    nbr, _ = SP.conv_table(c.to(cuda), c.to(cuda), BATCH, SHAPE, SHAPE, K3, S1, P1)
    assert torch.equal(nbr.cpu(), nbr_ref)
    w, scale, shift, g = _weights(n + cout, 27, 64, cout)
    res = torch.randn((n, cout), generator=g)
    args = dict(scale=scale, shift=shift, res=res, relu=True) if epilogue else {}
    ref, bound = _ref_conv(x, nbr_ref, w, **args)
    _check(_launch(cuda, x, nbr, w, prec, **args), ref, bound, prec, f"n={n}")


def test_restatement_is_the_oracle():
    """the float64 restatement used throughout this file is oracle.spconv_oracle.indice_conv"""
    feats, _ = _cloud()
    w, scale, shift, g = _weights(1, 27, 64, 64)
    res = torch.randn((300, 64), generator=g)
    ref, _ = _ref_conv(feats[:300, :64], _subm_table(300), w, scale, shift, res, True)
    assert torch.equal(ref.float(), SO.indice_conv(feats[:300, :64], _subm_table(300), w, scale, shift, res, True))


# ----------------------------------------------------------------------------------------------------------------------
# b. channel edges
# ----------------------------------------------------------------------------------------------------------------------
CH_FP32 = [(4, 4), (4, 64), (20, 36), (36, 68), (64, 132), (132, 64), (16, 260)]
CH_TC = [(64, 64), (64, 192), (128, 320), (192, 64), (320, 128), (64, 128), (128, 256)]


@pytest.mark.parametrize("cin,cout,prec", [(a, b, "fp32") for a, b in CH_FP32] + [(a, b, p) for a, b in CH_TC for p in ("bf16", "fp32_tc")])
def test_channel_edges(cuda, cin, cout, prec):
    n = 333   # two full 128-row tiles and a partial one; five 64-row tiles and a partial one
    x, nbr = _cloud()[0][:n, :cin], _subm_table(n)
    w, scale, shift, g = _weights(cin * 1000 + cout, 27, cin, cout)
    res = torch.randn((n, cout), generator=g)
    for args in ({}, dict(scale=scale, shift=shift, res=res, relu=True)):
        ref, bound = _ref_conv(x, nbr, w, **args)
        _check(_launch(cuda, x, nbr, w, prec, **args), ref, bound, prec, f"{cin}->{cout}")


# ----------------------------------------------------------------------------------------------------------------------
# c. kernel volumes and geometries, through the layer classes
# ----------------------------------------------------------------------------------------------------------------------
def _set(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.weight.copy_(torch.randn(m.weight.shape, generator=g) / (m.weight[..., 0, 0].numel() * m.in_channels) ** 0.5 * 2)
        if m.bias is not None:
            m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.3)
    return m


@pytest.mark.parametrize("prec", PRECS)
def test_conv1x1_forward_and_gradients(cuda, prec):
    """KV = 1: the conv1x1 branch of SparseConvolution.forward (its own arange table), with bias; forward, dX, dW, dbias"""
    from sst_b200 import spconv_modules as SP
    n = 700
    feats, coors = _cloud()
    x0, c = feats[:n, :64], coors[:n]
    m = _set(SP.SubMConv3d(64, 128, 1, bias=True), 3).to(cuda)
    m.precision = prec
    w, b = m.weight.detach().cpu().reshape(1, 64, 128), m.bias.detach().cpu()
    ident = torch.arange(n, dtype=torch.int32).view(-1, 1)
    ref, bound = _ref_conv(x0, ident, w, shift=b)
    with torch.no_grad():
        y = m(SP.SparseConvTensor(x0.to(cuda), c.to(cuda), SHAPE, BATCH))
    assert torch.equal(y.indices.cpu(), c) and y.spatial_shape == SHAPE
    _check(y.features, ref, bound, prec, "1x1 forward")
    x = x0.to(cuda).requires_grad_(True)
    y = m(SP.SparseConvTensor(x, c.to(cuda), SHAPE, BATCH)).features
    _check(y, ref, bound, prec, "1x1 forward (grad mode)")
    dy = torch.randn((n, 128), generator=torch.Generator().manual_seed(4))
    y.backward(dy.to(cuda))
    dx, bdx = _ref_dx(dy, ident, w, n)
    _check(x.grad, dx, bdx, prec, "1x1 dX")
    dw, bdw = _ref_dw(x0, ident, dy)
    assert bool(((m.weight.grad.double().cpu().reshape(1, 64, 128) - dw).abs() <= 1e-5 * bdw).all())
    torch.testing.assert_close(m.bias.grad.double().cpu(), dy.double().sum(0), rtol=1e-5, atol=1e-5 * float(dy.abs().sum(0).max()))


GEOMS = [((3, 1, 1), (2, 1, 1), (0, 0, 0)), ((2, 1, 1), (2, 1, 1), (0, 0, 0)), ((2, 2, 2), (2, 2, 2), (0, 0, 0)),
         ((3, 3, 3), (2, 2, 2), (0, 0, 0)), ((3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 3, 3), (2, 2, 2), (0, 1, 1))]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("ks,st,pd", GEOMS, ids=lambda v: "".join(map(str, v)))
def test_strided_then_inverse(cuda, ks, st, pd, prec):
    """KV 2, 3, 8, 27: SparseConv3d -> SparseInverseConv3d, coordinates bit-exact and features against float64 at both stages"""
    from sst_b200 import spconv_modules as SP
    n = 900
    feats, coors = _cloud()
    x, c = feats[:n, :64], coors[:n]
    conv = _set(SP.SparseConv3d(64, 64, ks, stride=st, padding=pd, bias=False, indice_key="k"), 5).to(cuda)
    inv = _set(SP.SparseInverseConv3d(64, 64, ks, indice_key="k", bias=False), 6).to(cuda)
    conv.precision = inv.precision = prec
    with torch.no_grad():
        y = conv(SP.SparseConvTensor(x.to(cuda), c.to(cuda), SHAPE, BATCH))
        z = inv(y)
    oc = SO.out_coors(c, BATCH, SHAPE, ks, st, pd)
    nbr = SO.neighbour_table(c, oc, BATCH, SHAPE, ks, st, pd)
    kv = nbr.shape[1]
    assert torch.equal(y.indices.cpu(), oc) and y.spatial_shape == SO.conv_output_size(SHAPE, ks, st, pd)
    ref_y, by = _ref_conv(x, nbr, conv.weight.detach().cpu().reshape(kv, 64, 64))
    _check(y.features, ref_y, by, prec, "strided")
    assert torch.equal(z.indices.cpu(), c) and z.spatial_shape == SHAPE
    ref_z, bz = _ref_conv(y.features.cpu(), _transpose_table(nbr, n), inv.weight.detach().cpu().reshape(kv, 64, 64))
    _check(z.features, ref_z, bz, prec, "inverse")
    # the float64 restatement of the pair is the oracle's dense one
    if prec == "fp32":
        dense_y, oc2, _ = SO.sparse_conv(x.double(), c, BATCH, SHAPE, conv.weight.detach().cpu().double(), st, pd)
        assert torch.equal(oc2, oc)
        torch.testing.assert_close(dense_y, ref_y, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("prec", PRECS)
def test_2d_layers(cuda, prec):
    """KV = 9, ndim == 2: SubMConv2d, SparseConv2d -> SparseInverseConv2d ((b, y, x) rows; the z column is added and dropped again)"""
    from sst_b200 import spconv_modules as SP
    g = torch.Generator().manual_seed(8)
    shape2, n = [36, 44], 500
    cells = torch.randperm(2 * 36 * 44, generator=g)[:n]
    c2 = torch.stack([cells // (36 * 44), cells % (36 * 44) // 44, cells % 44], 1).int()
    c3 = torch.cat([c2[:, :1], torch.zeros_like(c2[:, :1]), c2[:, 1:]], 1)
    x = torch.randn((n, 64), generator=g)
    sub = _set(SP.SubMConv2d(64, 64, 3, bias=True, indice_key="s"), 1).to(cuda)
    conv = _set(SP.SparseConv2d(64, 128, 3, stride=2, padding=1, bias=False, indice_key="k"), 2).to(cuda)
    inv = _set(SP.SparseInverseConv2d(128, 64, 3, indice_key="k", bias=False), 3).to(cuda)
    for m in (sub, conv, inv):
        m.precision = prec
    with torch.no_grad():
        a = sub(SP.SparseConvTensor(x.to(cuda), c2.to(cuda), shape2, 2))
        b = conv(a)
        z = inv(b)
    s3 = [1] + shape2
    nbr_s = SO.neighbour_table(c3, c3, 2, s3, [1, 3, 3], S1, [0, 1, 1])
    ref_a, ba = _ref_conv(x, nbr_s, sub.weight.detach().cpu().reshape(9, 64, 64), shift=sub.bias.detach().cpu())
    assert torch.equal(a.indices.cpu(), c2) and a.spatial_shape == shape2
    _check(a.features, ref_a, ba, prec, "SubMConv2d")
    oc = SO.out_coors(c3, 2, s3, [1, 3, 3], [1, 2, 2], [0, 1, 1])
    nbr = SO.neighbour_table(c3, oc, 2, s3, [1, 3, 3], [1, 2, 2], [0, 1, 1])
    assert torch.equal(b.indices.cpu(), oc[:, [0, 2, 3]]) and b.spatial_shape == [18, 22]
    ref_b, bb = _ref_conv(a.features.cpu(), nbr, conv.weight.detach().cpu().reshape(9, 64, 128))
    _check(b.features, ref_b, bb, prec, "SparseConv2d")
    ref_z, bz = _ref_conv(b.features.cpu(), _transpose_table(nbr, n), inv.weight.detach().cpu().reshape(9, 128, 64))
    assert torch.equal(z.indices.cpu(), c2) and z.spatial_shape == shape2
    _check(z.features, ref_z, bz, prec, "SparseInverseConv2d")


# ----------------------------------------------------------------------------------------------------------------------
# d. degenerate tables
# ----------------------------------------------------------------------------------------------------------------------
def _grid_rows(b, shape):
    z, y, x = torch.meshgrid(*[torch.arange(s) for s in shape], indexing="ij")
    return torch.stack([torch.full_like(z, b), z, y, x], -1).reshape(-1, 4)


def _corners(b, shape):
    return torch.tensor([[b, z, y, x] for z in (0, shape[0] - 1) for y in (0, shape[1] - 1) for x in (0, shape[2] - 1)])


def _degenerate(name):
    """(coors, batch_size, shape)"""
    g = torch.Generator().manual_seed(len(name))
    if name == "dense":          # every cell active: interior rows have all 27 neighbours, faces / edges / corners the exact subset
        shape, b = [5, 6, 7], 2
        c = torch.cat([_grid_rows(i, shape) for i in range(b)])
    elif name == "single":
        shape, b, c = [5, 6, 7], 1, torch.tensor([[0, 2, 3, 4]])
    elif name == "corners":      # the eight corners of the grid, in every sample
        shape, b = [5, 6, 7], 3
        c = torch.cat([_corners(i, shape) for i in range(b)])
    elif name == "empty_samples":   # a middle sample and the last sample hold nothing
        shape, b = [6, 12, 12], 4
        c = torch.cat([SO.synth_sparse(1, 1, shape, 150, 1)[1].long() + torch.tensor([i, 0, 0, 0]) for i in (0, 2)])
    else:                        # "one_sample": everything in sample 2 of 4
        shape, b = [6, 12, 12], 4
        c = SO.synth_sparse(2, 1, shape, 300, 1)[1].long() + torch.tensor([2, 0, 0, 0])
    return c[torch.randperm(c.shape[0], generator=g)].int(), b, shape


@pytest.mark.parametrize("name", ["dense", "single", "corners", "empty_samples", "one_sample"])
def test_degenerate_tables(cuda, name):
    from sst_b200 import spconv_modules as SP
    c, b, shape = _degenerate(name)
    n = c.shape[0]
    nbr_ref = SO.neighbour_table(c, c, b, shape, K3, S1, P1)
    nbr, inv = SP.conv_table(c.to(cuda), c.to(cuda), b, shape, shape, K3, S1, P1, want_nbr=True, want_inv=True)
    assert torch.equal(nbr.cpu(), nbr_ref) and torch.equal(inv.cpu(), _transpose_table(nbr_ref, n))
    if name == "dense":
        interior = ((c[:, 1:] > 0) & (c[:, 1:] < torch.tensor(shape) - 1)).all(1)
        assert bool((nbr_ref[interior] >= 0).all()) and int((nbr_ref >= 0).sum(1).min()) == 8
    if name in ("single", "corners"):
        assert int((nbr_ref >= 0).sum()) == n   # only the centre offset
    # strided tables on the same coordinates
    oshape = SO.conv_output_size(shape, K3, [2, 2, 2], P1)
    oc_ref = SO.out_coors(c, b, shape, K3, [2, 2, 2], P1)
    oc = SP.conv_out_coors(c.to(cuda), b, shape, oshape, K3, [2, 2, 2], P1)
    assert torch.equal(oc.cpu(), oc_ref)
    down, _ = SP.conv_table(c.to(cuda), oc, b, shape, oshape, K3, [2, 2, 2], P1)
    assert torch.equal(down.cpu(), SO.neighbour_table(c, oc_ref, b, shape, K3, [2, 2, 2], P1))
    x = torch.randn((n, 64), generator=torch.Generator().manual_seed(n))
    w, scale, shift, g = _weights(n, 27, 64, 64)
    ref, bound = _ref_conv(x, nbr_ref, w, scale, shift, None, True)
    for prec in PRECS:
        _check(_launch(cuda, x, nbr, w, prec, scale, shift, None, True), ref, bound, prec, name)


@pytest.mark.parametrize("prec", PRECS)
def test_tile_without_pairs(cuda, prec):
    """Inverse of a kernel (1,1,2) / stride (1,1,4) / padding 0 convolution: input cells with x % 4 in (2, 3) are covered by no output,
    so their rows of the inverse table are all -1.  Rows are ordered so that 128-row tile 1 holds only such rows (no stage at all: the
    output is the epilogue of zero), tile 2 only x % 4 == 0 rows (exactly one offset = one stage), tiles 0 and 3 a mixture."""
    from sst_b200 import spconv_modules as SP
    shape, ks, st, pd = [4, 16, 32], [1, 1, 2], [1, 1, 4], [0, 0, 0]
    g = torch.Generator().manual_seed(12)
    cells = _grid_rows(0, shape)
    cells = cells[torch.randperm(cells.shape[0], generator=g)]
    first, rest = cells[:128], cells[128:]
    cls = rest[:, 3] % 4
    c = torch.cat([first, rest[cls >= 2][:128], rest[cls == 0][:128], rest[cls == 1][:70]]).int()
    n = c.shape[0]
    oshape = SO.conv_output_size(shape, ks, st, pd)
    oc_ref = SO.out_coors(c, 1, shape, ks, st, pd)
    oc = SP.conv_out_coors(c.to(cuda), 1, shape, oshape, ks, st, pd)
    assert torch.equal(oc.cpu(), oc_ref)
    nbr_ref = SO.neighbour_table(c, oc_ref, 1, shape, ks, st, pd)
    inv_ref = _transpose_table(nbr_ref, n)
    nbr, inv = SP.conv_table(c.to(cuda), oc, 1, shape, oshape, ks, st, pd, want_nbr=True, want_inv=True)
    assert torch.equal(nbr.cpu(), nbr_ref) and torch.equal(inv.cpu(), inv_ref)
    assert bool((inv_ref[128:256] < 0).all()) and bool((inv_ref[256:384, 0] >= 0).all()) and bool((inv_ref[256:384, 1] < 0).all())
    y = torch.randn((oc_ref.shape[0], 64), generator=g)
    w, scale, shift, g2 = _weights(5, 2, 64, 128)
    res = torch.randn((n, 128), generator=g2)
    out = _launch(cuda, y, inv, w, prec, scale, shift, res, True)
    ref, bound = _ref_conv(y, inv_ref, w, scale, shift, res, True)
    _check(out, ref, bound, prec, "inverse with uncovered rows")
    assert torch.equal(out[128:256].cpu(), (shift + res[128:256]).clamp_min(0))   # the epilogue of zero, exactly
    _check(_launch(cuda, y, inv, w, prec), *_ref_conv(y, inv_ref, w), prec, "inverse with uncovered rows, no epilogue")


# ----------------------------------------------------------------------------------------------------------------------
# e. large key space
# ----------------------------------------------------------------------------------------------------------------------
def _sorted_table(coors, batch, shape, ks, st, pd, out_coors):
    """neighbour table by sorting linearised int64 keys (device tensors): no dense grid"""
    key = lambda c: ((c[:, 0].long() * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]
    skey, order = torch.sort(key(coors))
    cols = []
    for dz in range(ks[0]):
        for dy in range(ks[1]):
            for dx in range(ks[2]):
                q = out_coors.long().clone()
                q[:, 1] = q[:, 1] * st[0] - pd[0] + dz
                q[:, 2] = q[:, 2] * st[1] - pd[1] + dy
                q[:, 3] = q[:, 3] * st[2] - pd[2] + dx
                ok = ((q[:, 1:] >= 0) & (q[:, 1:] < torch.tensor(shape, device=q.device))).all(1)
                k = key(q)
                pos = torch.searchsorted(skey, k).clamp_max(skey.numel() - 1)
                hit = ok & (skey[pos] == k)
                cols.append(torch.where(hit, order[pos], torch.full_like(pos, -1)))
    return torch.stack(cols, 1).int()


@pytest.mark.parametrize("batch", [2, 24], ids=["B2", "B24_keys_beyond_2^31"])
def test_large_key_space(cuda, batch):
    """PartA2's grid [41, 1600, 1408]: ~20k voxels in the first and the last sample, the last cell of the last sample among them.
    B = 24 puts the linear keys of the last sample above 2^31 (2.2e9 cells; bitmap 277 MB + as much for its word prefix)."""
    from sst_b200 import spconv_modules as SP
    shape = [41, 1600, 1408]
    g = torch.Generator().manual_seed(batch)
    rows = []
    for b in (0, batch - 1):
        centre = torch.tensor([20, 800, 700]) if b == 0 else torch.tensor([40, 1598, 1406])
        pts = centre + (torch.randn((14000, 3), generator=g) * torch.tensor([2.0, 30.0, 30.0])).round().long()
        ok = ((pts >= 0) & (pts < torch.tensor(shape))).all(1)
        rows.append(torch.cat([torch.full((int(ok.sum()), 1), b), pts[ok]], 1))
    rows.append(torch.tensor([[batch - 1, 40, 1599, 1407], [batch - 1, 40, 1599, 1406], [0, 0, 0, 0]]))
    c = torch.unique(torch.cat(rows), dim=0)
    c = c[torch.randperm(c.shape[0], generator=g)].int().to(cuda)
    assert c.shape[0] > 12000
    nbr, inv = SP.conv_table(c, c, batch, shape, shape, K3, S1, P1, want_nbr=True, want_inv=True)
    ref = _sorted_table(c, batch, shape, K3, S1, P1, c)
    assert torch.equal(nbr, ref)
    assert torch.equal(inv, _transpose_table(ref.cpu(), c.shape[0]).to(cuda))
    last = int(torch.nonzero((c == torch.tensor([batch - 1, 40, 1599, 1407], device=cuda, dtype=torch.int32)).all(1))[0])
    assert int(nbr[last, 13]) == last and int(nbr[last, 12]) >= 0 and bool((nbr[last, 14:] < 0).all())
    # strided: output coordinates (sorted, unique) and the table onto them
    st, oshape = [2, 2, 2], SO.conv_output_size(shape, K3, [2, 2, 2], P1)
    oc = SP.conv_out_coors(c, batch, shape, oshape, K3, st, P1)
    cand = []
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                t = c.long().clone()
                t[:, 1:] += torch.tensor([1 - dz, 1 - dy, 1 - dx], device=cuda)
                ok = (t[:, 1:] >= 0).all(1) & (t[:, 1:] % 2 == 0).all(1)
                t[:, 1:] //= 2
                ok &= (t[:, 1:] < torch.tensor(oshape, device=cuda)).all(1)
                cand.append(t[ok])
    assert torch.equal(oc.long(), torch.unique(torch.cat(cand), dim=0))
    down, _ = SP.conv_table(c, oc, batch, shape, oshape, K3, st, P1)
    assert torch.equal(down, _sorted_table(c, batch, shape, K3, st, P1, oc))


# ----------------------------------------------------------------------------------------------------------------------
# f. backward at the edges
# ----------------------------------------------------------------------------------------------------------------------
def _check_dw(cuda, x, nbr, dy, what):
    """dW against float64, 1e-5 per element of the absolute-value bound; fp32 atomics across 1024-row chunks, so two runs agree to
    rounding (1e-6 of the bound), not bit for bit"""
    from sst_b200 import spconv_modules as SP
    kv, cin, cout = nbr.shape[1], x.shape[1], dy.shape[1]
    ref, mag = _ref_dw(x, nbr, dy)
    a = SP.indice_conv_backward_weight(x.to(cuda), nbr.to(cuda), dy.to(cuda), kv, cin, cout)
    b = SP.indice_conv_backward_weight(x.to(cuda), nbr.to(cuda), dy.to(cuda), kv, cin, cout)
    err = (a.double().cpu() - ref).abs()
    worst = torch.argmax(err - 1e-5 * mag)
    assert bool((err <= 1e-5 * mag).all()), f"{what}: dW element {int(worst)} off by {float(err.flatten()[worst]):.3e} (bound {float(mag.flatten()[worst]):.3e})"
    assert bool(((a - b).abs().double().cpu() <= 1e-6 * mag).all()), f"{what}: two runs differ beyond rounding"


@pytest.mark.parametrize("cin,cout", [(4, 4), (20, 36), (64, 64), (64, 132), (128, 64)])
@pytest.mark.parametrize("n", [1, 127, 129, 1023, 1024, 1025, 2049, 3000])
def test_weight_gradient_edges(cuda, n, cin, cout):
    x, nbr = _cloud()[0][:n, :cin], _subm_table(n)
    dy = torch.randn((n, cout), generator=torch.Generator().manual_seed(n + cout))
    _check_dw(cuda, x, nbr, dy, f"n={n} {cin}->{cout}")


def test_weight_gradient_chunk_without_pairs(cuda):
    """offsets 0 and 13 have no pair inside the second 1024-row chunk (its CTAs return before the reduction); the other chunks do"""
    n = 3000
    nbr = _subm_table(n).clone()
    nbr[1024:2048, 0] = -1
    nbr[1024:2048, 13] = -1
    assert bool((nbr[:1024, 0] >= 0).any()) and bool((nbr[2048:, 0] >= 0).any())
    x = _cloud()[0][:n, :64]
    dy = torch.randn((n, 64), generator=torch.Generator().manual_seed(2))
    _check_dw(cuda, x, nbr, dy, "empty chunk")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("kind", ["subm", "strided", "inverse"])
@pytest.mark.parametrize("n", [129, 1025])
def test_input_gradient(cuda, n, kind, prec):
    """dX through _IndiceConvFunction (the forward kernel on the transposed table with W^T) against float64"""
    from sst_b200 import spconv_modules as SP
    feats, coors = _cloud()
    x0, c = feats[:n, :64], coors[:n]
    ks, st, pd = K3, [2, 2, 2], [0, 1, 1]
    g = torch.Generator().manual_seed(n)
    if kind == "subm":
        layers = [_set(SP.SubMConv3d(64, 128, 3, bias=False, indice_key="s"), 1)]
        nbr = _subm_table(n)
    else:
        layers = [_set(SP.SparseConv3d(64, 128, ks, stride=st, padding=pd, bias=False, indice_key="k"), 1)]
        oc = SO.out_coors(c, BATCH, SHAPE, ks, st, pd)
        nbr = SO.neighbour_table(c, oc, BATCH, SHAPE, ks, st, pd)
        if kind == "inverse":
            layers.append(_set(SP.SparseInverseConv3d(128, 64, ks, indice_key="k", bias=False), 2))
    for m in layers:
        m.to(cuda)
        m.precision = prec
    x = x0.to(cuda).requires_grad_(True)
    t = SP.SparseConvTensor(x, c.to(cuda), SHAPE, BATCH)
    if kind == "inverse":   # gradient w.r.t. the inverse layer's own input
        with torch.no_grad():
            mid = layers[0](t)
        xin = mid.features.clone().requires_grad_(True)
        out = layers[1](mid.replace_feature(xin)).features
        table, w, n_in, leaf = _transpose_table(nbr, n), layers[1].weight, xin.shape[0], xin
    else:
        out = layers[0](t).features
        table, w, n_in, leaf = nbr, layers[0].weight, n, x
    dy = torch.randn(out.shape, generator=g)
    out.backward(dy.to(cuda))
    dx, bound = _ref_dx(dy, table, w.detach().cpu().reshape(27, w.shape[-2], w.shape[-1]), n_in)
    _check(leaf.grad, dx, bound, prec, f"dX {kind}")
    dw, mag = _ref_dw(leaf.detach().cpu(), table, dy)
    assert bool(((w.grad.double().cpu().reshape(dw.shape) - dw).abs() <= 1e-5 * mag).all())


# ----------------------------------------------------------------------------------------------------------------------
# g. operand scale: the tolerance at 2^s is the tolerance at 1
# ----------------------------------------------------------------------------------------------------------------------
S_ACT = (-40, -30, -24, -20, -16, -12, -8, 0, 8, 14, 20, 30)
S_WGT = (-30, -20, -12, -8, 0, 8, 14)
N_SCALE = 700


@functools.lru_cache(maxsize=None)
def _scale_case():
    x, nbr = _cloud()[0][:N_SCALE, :64], _subm_table(N_SCALE)
    w = _weights(9, 27, 64, 64)[0]
    return (x, nbr, w) + _ref_conv(x, nbr, w)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("s", S_ACT)
def test_scale_features(cuda, s, prec):
    x, nbr, w, ref, bound = _scale_case()
    out = _launch(cuda, x * 2.0 ** s, nbr, w, prec)
    _check(out, ref * 2.0 ** s, bound * 2.0 ** s, prec, f"features x 2^{s}")
    assert torch.equal(out, _launch(cuda, x, nbr, w, prec) * 2.0 ** s)   # power-of-two scaling commutes with every rounding


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("s", S_WGT)
def test_scale_weights(cuda, s, prec):
    x, nbr, w, ref, bound = _scale_case()
    out = _launch(cuda, x, nbr, w * 2.0 ** s, prec)
    _check(out, ref * 2.0 ** s, bound * 2.0 ** s, prec, f"weights x 2^{s}")
    assert torch.equal(out, _launch(cuda, x, nbr, w, prec) * 2.0 ** s)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("s", S_ACT)
def test_scale_grad_out(cuda, s, prec):
    """dX with grad_out x 2^s through autograd: rows of 1e-5 ... 1e-12 are what a mean-reduced loss hands the backward"""
    from sst_b200 import spconv_modules as SP
    x0, nbr, w, _, _ = _scale_case()
    c = _cloud()[1][:N_SCALE]
    m = SP.SubMConv3d(64, 64, 3, bias=False, indice_key="s").to(cuda)
    m.precision = prec
    with torch.no_grad():
        m.weight.copy_(w.reshape(3, 3, 3, 64, 64))
    x = x0.to(cuda).requires_grad_(True)
    out = m(SP.SparseConvTensor(x, c.to(cuda), SHAPE, BATCH)).features
    dy = torch.randn(out.shape, generator=torch.Generator().manual_seed(3))
    out.backward((dy * 2.0 ** s).to(cuda))
    dx, bound = _ref_dx(dy, nbr, w, N_SCALE)
    _check(x.grad, dx * 2.0 ** s, bound * 2.0 ** s, prec, f"grad_out x 2^{s}")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("table", ["subm27", "rows1"])
def test_scale_mixed_rows(cuda, table, prec):
    """Feature rows spanning 2^-20 ... 2^8 in one tensor.  The exponent is per OUTPUT row (the smallest among the rows it gathers), so
    every output row meets the unit-scale tolerance relative to its own absolute-value bound: with KV = 1 that is every row relative
    to itself; with KV = 27 a small row next to a large one is rounded relative to the large one, which dominates the bound of every
    output both reach."""
    x, nbr, w, _, _ = _scale_case()
    u = torch.randint(-20, 9, (N_SCALE, 1), generator=torch.Generator().manual_seed(6)).double()
    x = (x.double() * 2.0 ** u).float()
    if table == "rows1":
        nbr, w = torch.arange(N_SCALE, dtype=torch.int32).view(-1, 1), w[13:14]
    ref, bound = _ref_conv(x, nbr, w)
    out = _launch(cuda, x, nbr, w, prec).double().cpu()
    err = (out - ref).abs().amax(1)
    assert bool((err <= ROW_TOL[prec] * bound).all()), f"worst row ratio {float((err / bound).max()):.2e}"
    assert float(bound.min()) < 2.0 ** -12 * float(bound.max())   # the case does hold rows of very different size


# ----------------------------------------------------------------------------------------------------------------------
# h. caches that outlive a flat-buffer update
# ----------------------------------------------------------------------------------------------------------------------
def _ref_block(net, x, nbr):
    conv, bn = net[0], net[1]
    sd = {k: v.detach().double().cpu() for k, v in bn.state_dict().items()}
    scale = sd["weight"] / torch.sqrt(sd["running_var"] + bn.eps)
    return _ref_conv(x, nbr, conv.weight.detach().cpu().reshape(27, 64, 64), scale, sd["bias"] - sd["running_mean"] * scale, None, True)


@pytest.mark.parametrize("prec", PRECS)
def test_caches_follow_flat_buffer_updates(cuda, prec):
    """eval-mode SubMConv3d + BatchNorm1d + ReLU (one fused launch over the cached 16-bit weights and folded BatchNorm) stays right
    after FlatAdamW.step, after a write to the optimizer's flat buffer and after load_state_dict"""
    from sst_b200 import spconv_modules as SP
    from sst_b200.train import FlatAdamW
    n = 500
    x, c, nbr = _cloud()[0][:n, :64], _cloud()[1][:n], _subm_table(n)
    torch.manual_seed(3)
    net = SP.SparseSequential(SP.SubMConv3d(64, 64, 3, bias=False, indice_key="s"), torch.nn.BatchNorm1d(64), torch.nn.ReLU()).to(cuda).eval()
    with torch.no_grad():
        net[1].running_mean.normal_(0, 0.2)
        net[1].running_var.uniform_(0.5, 1.5)
        net[1].weight.uniform_(0.5, 1.5)
        net[1].bias.normal_(0, 0.2)
    SP.set_spconv_precision(net, prec)

    def run_and_check(what):
        with torch.no_grad():
            out = net(SP.SparseConvTensor(x.to(cuda), c.to(cuda), SHAPE, BATCH)).features
        _check(out, *_ref_block(net, x, nbr), prec, what)
        return out

    first = run_and_check("fresh")
    opt = FlatAdamW(list(net.parameters()), lr=0.05, weight_decay=0.0)
    run_and_check("parameters moved into the flat buffer")
    opt.flat_grad.normal_()
    opt.step()
    stepped = run_and_check("after FlatAdamW.step")
    assert float((stepped - first).abs().max()) > 1e-2 * float(first.abs().max())   # the step did move the output
    opt.flat.mul_(0.5)
    run_and_check("after an in-place write to the flat buffer")
    sd = {k: (v * 1.5 if v.dtype.is_floating_point else v) for k, v in net.state_dict().items()}
    net.load_state_dict(sd)
    run_and_check("after load_state_dict")
