"""GPU: the voxel index layer (csrc/index.cuh: bitmap-rank unique rows, CSR grouping, segmented reduce, stable in-group rank) against
float64 on every dispatch route, grid size and segment edge, through the entry points of csrc/voxel.cu.

`launch_segment_reduce` picks one of ten kernels from the channel count C and the alignment of the rows:
    v4  (GROUP, NV4)   C % 4 == 0, C <= 256, src / out / argmax 16-byte aligned; GROUP lanes per segment, NV4 float4 per lane,
                       RIF rows in flight per lane (8 for NV4 = 1, 4 for NV4 = 2); ARG = argmax wanted (else one fmaxf per element)
        1,1  C = 4             2,1  C = 8             4,1  C = 12, 16        8,1  C = 20, 32
        16,1 C = 36, 64        32,1 C = 68, 128       32,2 C = 132, 256
    scalar GROUP       every other case
        4    C = 1, 2, 3       8    C = 5, 7, 31      32   C = 33, 65, 260, 300
    scalar, misaligned C % 4 == 0 with src a view at a storage offset of one float: C = 4 (GROUP 4), 8 (8), 64 and 132 (32)
Each route runs through `ops.segment_reduce` (sum, mean, max with argmax, max without) and `ops.dynamic_point_to_voxel_forward`
(sum, mean, max) and its backward, on segments of 1, GROUP - 1, GROUP, GROUP + 1 and 2 GROUP + 1 rows, on sizes that end inside a batch
of RIF rows, on empty segments (gaps in the index and num_segments past max(index) + 1) and, in test_one_segment_holds_every_point, on
one segment of 200 000 rows.  Rows are shuffled, so the CSR order inside a segment is arbitrary.

`launch_mark_rows` / `launch_emit_rows` pick their path from the grid size T (cells of the bounding box of the rows):
    T <= 393 216                 block-private bitmap in at most 48 KB of shared memory
    393 216 < T <= 786 432       the same in opt-in shared memory (up to 96 KB)
    T > 786 432                  global bitmap, one test-and-atomicOr per row
    T >= 2^31                    64-bit key decode in emit_rows (the grid of decode64 puts keys above 2^32)
    T > 2^34                     SSTB_ERR_UNSUPPORTED (-3), nothing launched
They run through `ops.unique_rows` (k = 1..4 columns, negative lower bounds), dynamic scatter and `ops.get_inner_win_inds`, with
T % 32 in {0, 1, 31} and rows on the first and the last cell.

Reference: oracle.sst_oracle (dynamic_point_to_voxel_forward / backward, segment_reduce, ingroup_indices, dynamic_voxelize,
voxelize_with_batch_idx) on float64 inputs, torch.unique(dim=0) for rows; for max, the row attaining it is the lowest row index among
the rows equal to the max, and the value (sign of a zero included) is that row's.  When oracle/_ref holds the reference's own voxel
layer, dynamic scatter forward and backward are also compared with it (test_dynamic_scatter_vs_reference_cuda).

Bounds:
    coordinates, inverse map, counts, voxel count, argmax, max values, in-group ranks, voxel coordinates   bit-exact
    sum    |got - ref| <= 2^-24 |ref| + 2^-50 sum|x|        per output element (fp64 accumulation, one fp32 rounding)
    mean   |got - ref| <= 2^-23 |ref| + 2^-50 sum|x| / n    (two fp32 roundings)
    dyadic features spanning less than 2^29 (test_exact_sums): the fp64 sum is exact, so sum == float(exact) and
           mean == float(float(exact) / n), bit for bit
    backward of dynamic scatter: bit-exact (sum copies, mean is one IEEE division on both sides, max sends the gradient to the lowest
           row attaining the max); backward of segment_reduce max: the whole gradient to the argmax row.
Max on the plain fmaxf route (no argmax) is compared with == only: fmaxf does not specify which zero it returns for (+0, -0).  NaN
propagation is not pinned; the argmax and the plain route must only agree on it.  Rows whose segment index lies outside
[0, num_segments) are dropped, forward and backward.  Every route is called twice and must give bit-identical outputs."""
import math

import numpy as np
import pytest
import torch

from oracle import build_ref, sst_oracle as O

pytestmark = pytest.mark.gpu

V4_C = (4, 8, 12, 16, 20, 32, 36, 64, 68, 128, 132, 256)
SCALAR_C = (1, 2, 3, 5, 7, 31, 33, 65, 260, 300)
MISALIGNED_C = (4, 8, 64, 132)
ROUTES = [(c, False) for c in V4_C + SCALAR_C] + [(c, True) for c in MISALIGNED_C]
GRID = (20, 30, 40)  # (z, y, x) cells of the dynamic-scatter cases


def _route(C, misaligned):
    """(name, GROUP, RIF) of launch_segment_reduce for C channels"""
    if C % 4 == 0 and C <= 256 and not misaligned:
        c4 = C // 4
        G, nv4 = next(gv for lim, gv in ((32, (32, 2)), (16, (32, 1)), (8, (16, 1)), (4, (8, 1)), (2, (4, 1)), (1, (2, 1)), (0, (1, 1)))
                      if c4 > lim)
        return f"v4_{G}x{nv4}", G, 8 if nv4 == 1 else 4
    G = 32 if C >= 32 else 8 if C > 4 else 4
    return f"scalar_{G}" + ("_misaligned" if misaligned else ""), G, 8


ROUTE_IDS = [f"C{c}-{_route(c, m)[0]}" for c, m in ROUTES]
assert [_route(c, False)[0] for c in (4, 8, 12, 16, 20, 32, 36, 64, 68, 128, 132, 256)] == [
    "v4_1x1", "v4_2x1", "v4_4x1", "v4_4x1", "v4_8x1", "v4_8x1", "v4_16x1", "v4_16x1", "v4_32x1", "v4_32x1", "v4_32x2", "v4_32x2"]


def _edge_sizes(C, misaligned):
    """segment sizes on the route's edges: 1, GROUP +- 1, GROUP, 2 GROUP + 1 and sizes that end inside a batch of RIF rows"""
    _, G, rif = _route(C, misaligned)
    s = {1, G - 1, G, G + 1, 2 * G + 1, rif - 1, rif + 1, 2 * rif + 3, G + rif // 2 + 1, 3 * G + rif - 1}
    return sorted(v for v in s if v > 0)


def _segment_index(g, sizes, extra=150, extra_max=40):
    """index [P] int64 of segments with the given sizes plus `extra` random ones, rows shuffled; the segment ids leave gaps (empty
    segments), and num_segments = max id + 3 adds two empty segments at the end"""
    sizes = list(sizes) + torch.randint(1, extra_max + 1, (extra,), generator=g).tolist()
    n = len(sizes)
    ids = torch.sort(torch.randperm(n + n // 4 + 2, generator=g)[:n]).values
    index = torch.repeat_interleave(ids, torch.tensor(sizes))
    return index[torch.randperm(index.numel(), generator=g)].contiguous(), int(ids.max()) + 3


def _voxel_coors(g, sizes, invalid):
    """coors [P, 3] int32 (z, y, x): one distinct GRID cell per size with that many rows, and `invalid` rows with a negative
    coordinate in one random column; rows shuffled"""
    cells = torch.randperm(GRID[0] * GRID[1] * GRID[2], generator=g)[:len(sizes)]
    zyx = torch.stack([cells // (GRID[1] * GRID[2]), cells // GRID[2] % GRID[1], cells % GRID[2]], 1)
    co = zyx.repeat_interleave(torch.tensor(sizes), 0)
    if invalid:
        bad = torch.randint(0, min(GRID), (invalid, 3), generator=g)
        bad[torch.arange(invalid), torch.randint(0, 3, (invalid,), generator=g)] = -torch.randint(1, 4, (invalid,), generator=g)
        co = torch.cat([co, bad])
    return co[torch.randperm(co.shape[0], generator=g)].to(torch.int32).contiguous()


def _randn(g, P, C):
    return (torch.randn(P, C, generator=g) * 8).float()


def _device_rows(x, dev, misaligned):
    """x on the device; misaligned: a contiguous view at a storage offset of one float (rows no longer 16-byte aligned)"""
    if not misaligned:
        return x.to(dev)
    buf = torch.empty(x.numel() + 1, dtype=torch.float32, device=dev)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4
    return v


def _same_bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _keep(index, nseg):
    return (index >= 0) & (index < nseg)


def _ref_sum(x64, index, nseg):
    """float64 sum, sum of |x| and row count of every segment, over the rows whose index lies in [0, nseg)"""
    k = _keep(index, nseg)
    idx, v = index[k], x64[k]
    return (O.segment_reduce(v, idx, "sum", nseg), O.segment_reduce(v.abs(), idx, "sum", nseg), torch.bincount(idx, minlength=nseg))


def _ref_max(x64, index, nseg):
    """(value, argmax) of the max over the in-range rows: argmax = the lowest row index among the rows equal to the max, value = that
    row's (so the sign of a zero is the lowest row's); an empty segment gives 0 and P"""
    P, C = x64.shape
    k = _keep(index, nseg)
    rows, idx, v = torch.arange(P)[k], index[k], x64[k]
    ix = idx[:, None].expand(-1, C)
    mx = torch.full((nseg, C), -math.inf, dtype=torch.float64).scatter_reduce(0, ix, v, "amax", include_self=True)
    cand = torch.where(v == mx[idx], rows[:, None].expand(-1, C), P)
    arg = torch.full((nseg, C), P, dtype=torch.int64).scatter_reduce(0, ix, cand, "amin", include_self=True)
    val = torch.where(arg < P, x64.gather(0, arg.clamp(max=P - 1)), torch.zeros((), dtype=torch.float64))
    return val, arg


def _assert_within(got, ref, abssum, cnt, mode, what=""):
    """the sum / mean bound of the module docstring, per output element"""
    got = got.detach().cpu().double()
    assert got.shape == ref.shape
    if mode == "sum":
        bound = 2.0 ** -24 * ref.abs() + 2.0 ** -50 * abssum
    else:
        bound = 2.0 ** -23 * ref.abs() + 2.0 ** -50 * abssum / cnt.clamp(min=1).double()[:, None]
    bad = ~((got - ref).abs() <= bound)
    if bad.any():
        s, c = [int(t[0]) for t in torch.nonzero(bad, as_tuple=True)]
        raise AssertionError(f"{what} {mode}: {int(bad.sum())} of {bad.numel()} elements outside the bound; first at segment {s} "
                             f"channel {c}: got {got[s, c].item()!r}, float64 {ref[s, c].item()!r}, bound {bound[s, c].item():.3g}")


def _check_segment_reduce(ops, src, index, nseg, x, mode, cuda, what=""):
    """one route of ops.segment_reduce, run twice; mode in sum, mean, max (with argmax), max_noarg"""
    red = "max" if mode.startswith("max") else mode
    idx = index.to(cuda)
    (out, arg), (out2, arg2) = [ops.segment_reduce(src, idx, red, nseg, want_argmax=mode == "max") for _ in range(2)]
    assert _same_bits(out, out2) and (arg is None or torch.equal(arg, arg2)), f"{what}: two calls differ"
    if red == "max":
        val, ref_arg = _ref_max(x.double(), index, nseg)
        if mode == "max":
            assert torch.equal(arg.cpu(), ref_arg), f"{what}: argmax"
            assert _same_bits(out, val.float()), f"{what}: max values (sign bits included)"
        else:
            assert arg is None and torch.equal(out.cpu(), val.float()), f"{what}: max values"
    else:
        s, a, n = _ref_sum(x.double(), index, nseg)
        _assert_within(out, s if mode == "sum" else s / n.clamp(min=1).double()[:, None], a, n, mode, what)
    return out, arg


def _check_dynamic_scatter(ops, f, coors, x, mode, cuda, grad_seed, what=""):
    """ops.dynamic_point_to_voxel_forward (twice) and _backward against the oracle; returns the forward outputs"""
    co = coors.to(cuda)
    runs = [ops.dynamic_point_to_voxel_forward(f, co, mode) for _ in range(2)]
    g_f, g_c, g_m, g_n = runs[0]
    assert _same_bits(g_f, runs[1][0]) and all(torch.equal(a, b) for a, b in zip(runs[0][1:], runs[1][1:])), f"{what}: two calls differ"
    r_f, r_c, r_m, r_n = O.dynamic_point_to_voxel_forward(x.double(), coors, mode)
    assert torch.equal(g_c.cpu(), r_c) and torch.equal(g_m.cpu(), r_m) and torch.equal(g_n.cpu(), r_n), f"{what}: index outputs"
    if mode == "max":
        assert torch.equal(g_f.cpu(), r_f.float()), f"{what}: max values"
    else:
        a = O.dynamic_point_to_voxel_forward(x.double().abs(), coors, "sum")[0]
        _assert_within(g_f, r_f, a, r_n.long(), mode, what)
    gr = _randn(torch.Generator().manual_seed(grad_seed), r_f.shape[0], r_f.shape[1])
    grads = []
    for _ in range(2):
        gf = torch.full(f.shape, float("nan"), device=cuda)
        ops.dynamic_point_to_voxel_backward(gf, gr.to(cuda), f, g_f, g_m, g_n, mode)
        grads.append(gf)
    ref = O.dynamic_point_to_voxel_backward(gr.double(), x.double(), r_f, r_m, r_n, mode).float()
    assert _same_bits(grads[0], grads[1]), f"{what}: two backward calls differ"
    assert _same_bits(grads[0], ref), f"{what}: backward"
    return g_f, g_c, g_m, g_n


# ----------------------------------------------------------------------------------------------------------------------
# segmented reduce: every route
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["sum", "mean", "max", "max_noarg"])
@pytest.mark.parametrize("C,misaligned", ROUTES, ids=ROUTE_IDS)
def test_segment_reduce_routes(cuda, C, misaligned, mode):
    from sst_b200 import ops
    g = torch.Generator().manual_seed(1000 * C + misaligned)
    index, nseg = _segment_index(g, _edge_sizes(C, misaligned), extra_max=3 * _route(C, misaligned)[1] + 8)
    x = _randn(g, index.numel(), C)
    _check_segment_reduce(ops, _device_rows(x, cuda, misaligned), index, nseg, x, mode, cuda, ROUTE_IDS[ROUTES.index((C, misaligned))])


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
@pytest.mark.parametrize("C,misaligned", ROUTES, ids=ROUTE_IDS)
def test_dynamic_scatter_routes(cuda, C, misaligned, mode):
    """forward and backward; odd C has invalid rows (the (-1,-1,-1) row is dropped), even C has none (the first voxel is dropped)"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(2000 * C + misaligned)
    sizes = _edge_sizes(C, misaligned) + torch.randint(1, 3 * _route(C, misaligned)[1] + 9, (120,), generator=g).tolist()
    coors = _voxel_coors(g, sizes, invalid=9 if C % 2 else 0)
    x = _randn(g, coors.shape[0], C)
    _check_dynamic_scatter(ops, _device_rows(x, cuda, misaligned), coors, x, mode, cuda, C, ROUTE_IDS[ROUTES.index((C, misaligned))])


@pytest.mark.parametrize("C,misaligned", ROUTES, ids=ROUTE_IDS)
def test_exact_sums(cuda, C, misaligned):
    """dyadic features (integers below 2^10 times 2^k, k in [-14, 3]): the fp64 sums are exact, so sum == float(exact) and
    mean == float(float(exact) / n) bit for bit, through segment_reduce and dynamic scatter"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(3000 * C + misaligned)
    index, nseg = _segment_index(g, _edge_sizes(C, misaligned), extra=60, extra_max=3 * _route(C, misaligned)[1] + 8)
    dyadic = lambda P: (torch.randint(-1023, 1024, (P, C), generator=g) *  # noqa: E731
                        torch.pow(2.0, torch.randint(-14, 4, (P, C), generator=g))).float()
    x = dyadic(index.numel())
    exact, _, n = _ref_sum(x.double(), index, nseg)
    src = _device_rows(x, cuda, misaligned)
    s = ops.segment_reduce(src, index.to(cuda), "sum", nseg)[0]
    m = ops.segment_reduce(src, index.to(cuda), "mean", nseg)[0]
    assert _same_bits(s, exact.float())
    assert _same_bits(m, exact.float() / n.clamp(min=1).float()[:, None])
    coors = _voxel_coors(g, torch.randint(1, 40, (80,), generator=g).tolist(), invalid=5)
    x = dyadic(coors.shape[0])
    f = _device_rows(x, cuda, misaligned)
    r_sum, _, _, r_n = O.dynamic_point_to_voxel_forward(x.double(), coors, "sum")
    assert _same_bits(ops.dynamic_point_to_voxel_forward(f, coors.to(cuda), "sum")[0], r_sum.float())
    assert _same_bits(ops.dynamic_point_to_voxel_forward(f, coors.to(cuda), "mean")[0], r_sum.float() / r_n.float()[:, None])


@pytest.mark.parametrize("C", [1, 16, 132])
def test_one_segment_holds_every_point(cuda, C):
    """200 000 rows in one segment (and two empty ones after it), and the same rows in one voxel next to invalid rows"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(4000 + C)
    P = 200_000
    x = _randn(g, P, C)
    index = torch.zeros(P, dtype=torch.int64)
    src = x.to(cuda)
    for mode in ("sum", "mean", "max", "max_noarg"):
        _check_segment_reduce(ops, src, index, 3, x, mode, cuda, f"C{C}")
    coors = torch.full((P, 3), 2, dtype=torch.int32)
    coors[::997] = torch.tensor([-1, 4, 4], dtype=torch.int32)
    for mode in ("sum", "mean", "max"):
        out = _check_dynamic_scatter(ops, src, coors, x, mode, cuda, C, f"C{C}")
        assert out[0].shape[0] == 1


# ----------------------------------------------------------------------------------------------------------------------
# max: ties, signed zeros, -inf segments, extreme values, NaN
# ----------------------------------------------------------------------------------------------------------------------
EXTREMES = np.array([3.0e38, -3.0e38, np.finfo(np.float32).max, -np.finfo(np.float32).max, 2.9e38, 1e-45, -1e-45, 2e-40, -2e-40,
                     np.finfo(np.float32).tiny, -np.finfo(np.float32).tiny, 0.0, -0.0, 1.0], dtype=np.float32)


@pytest.mark.parametrize("data", ["integers", "extremes"])
@pytest.mark.parametrize("C", [3, 4, 8, 36, 132, 300])
def test_max_ties(cuda, C, data):
    """integer-valued ties (zeros of both signs among them) or values near +-3e38 and subnormals, and segments that are entirely -inf:
    forward and backward of segment_reduce (argmax and plain route) and of dynamic scatter"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(5000 + C + (data == "extremes"))
    index, nseg = _segment_index(g, _edge_sizes(C, False), extra=80, extra_max=20)
    P = index.numel()
    if data == "integers":
        x = torch.randint(-2, 3, (P, C), generator=g).float()
    else:
        x = torch.from_numpy(EXTREMES)[torch.randint(0, len(EXTREMES), (P, C), generator=g)]
    x[(x == 0) & (torch.rand(P, C, generator=g) < 0.5)] = -0.0
    x[index % 7 == 3] = -math.inf
    assert (torch.signbit(x) & (x == 0)).any() and (~torch.signbit(x) & (x == 0)).any()
    src = x.to(cuda)
    _check_segment_reduce(ops, src, index, nseg, x, "max_noarg", cuda, "plain")
    out, arg = _check_segment_reduce(ops, src, index, nseg, x, "max", cuda, "argmax")
    # backward of segment_reduce max: the whole gradient goes to the argmax row
    gout = _randn(g, nseg, C)
    leaf = src.clone().requires_grad_(True)
    o, a = ops.segment_reduce(leaf, index.to(cuda), "max", nseg)
    o.backward(gout.to(cuda))
    ref = torch.zeros(P + 1, C).scatter_(0, a.cpu(), gout)[:P]
    assert torch.equal(a.cpu(), arg.cpu()) and _same_bits(leaf.grad, ref)
    # dynamic scatter: the same rows grouped by voxel
    coors = _voxel_coors(g, torch.randint(1, 24, (60,), generator=g).tolist(), invalid=4)
    xs = x.repeat((coors.shape[0] + P - 1) // P, 1)[:coors.shape[0]].contiguous()
    _check_dynamic_scatter(ops, xs.to(cuda), coors, xs, "max", cuda, C, "dynamic scatter")


@pytest.mark.parametrize("C", [4, 5, 132])
def test_max_nan_routes_agree(cuda, C):
    """NaN propagation is not pinned; the argmax route and the plain route give the same values"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(6000 + C)
    index, nseg = _segment_index(g, _edge_sizes(C, False), extra=40)
    x = _randn(g, index.numel(), C) + 0.5
    x[torch.rand(x.shape, generator=g) < 0.2] = float("nan")
    x[index == index[0]] = float("nan")
    src, idx = x.to(cuda), index.to(cuda)
    a = ops.segment_reduce(src, idx, "max", nseg, want_argmax=True)[0]
    b = ops.segment_reduce(src, idx, "max", nseg, want_argmax=False)[0]
    assert _same_bits(a, b)


# ----------------------------------------------------------------------------------------------------------------------
# rows outside [0, num_segments)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [4, 5, 132])
def test_segment_reduce_drops_out_of_range_rows(cuda, C):
    """indices -2^40, -1, num_segments, num_segments + 1 and 2^40 contribute nothing, forward and backward"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(7000 + C)
    index, nseg = _segment_index(g, _edge_sizes(C, False), extra=60)
    P = index.numel()
    far = torch.tensor([-2 ** 40, -1, nseg, nseg + 1, nseg + 7, 2 ** 40])
    pick = torch.rand(P, generator=g) < 0.2
    index[pick] = far[torch.randint(0, len(far), (int(pick.sum()),), generator=g)]
    x = _randn(g, P, C)
    src, idx = x.to(cuda), index.to(cuda)
    for mode in ("sum", "mean", "max", "max_noarg"):
        _check_segment_reduce(ops, src, index, nseg, x, mode, cuda, mode)
    keep = _keep(index, nseg)
    k_idx = torch.where(keep, index, 0)
    gout = _randn(g, nseg, C)
    for mode in ("sum", "mean", "max"):
        leaf = src.clone().requires_grad_(True)
        out, arg = ops.segment_reduce(leaf, idx, mode, nseg)
        out.backward(gout.to(cuda))
        if mode == "max":
            ref = torch.zeros(P + 1, C).scatter_(0, arg.cpu(), gout)[:P]
        else:
            ref = torch.where(keep[:, None], gout[k_idx], 0.0)
            if mode == "mean":
                ref = ref / torch.bincount(index[keep], minlength=nseg).clamp(min=1)[k_idx].float()[:, None]
        assert _same_bits(leaf.grad, ref), mode
    # scatter_v2 with a caller's inverse and too few output rows: the rows of the missing ones are dropped
    coors = torch.randint(0, 9, (P, 2), generator=g)
    new_coors, inv = torch.unique(coors, dim=0, return_inverse=True)
    short = new_coors.shape[0] - 5
    out, _, _ = ops.scatter_v2(src, coors.to(cuda), "sum", unq_inv=inv.to(cuda), new_coors=new_coors[:short].to(cuda))
    s, a, n = _ref_sum(x.double(), inv, short)
    _assert_within(out, s, a, n, "sum", "scatter_v2")


# ----------------------------------------------------------------------------------------------------------------------
# bitmap-rank index: grid sizes
# ----------------------------------------------------------------------------------------------------------------------
INDEX_GRIDS = {  # per-column extents; T = their product
    "smem_k1_T%32=0": (32000,),
    "smem_k2_T%32=1": (33, 97),
    "optin_k3_T%32=31": (3, 11, 15999),
    "global_k4_T%32=0": (2, 3, 11, 16000),
    "global_k4_T%32=1": (3, 11, 3, 9611),
    "global_k1_T%32=31": (1000031,),
    "decode64_k3": (5, 40000, 30000),
}
for _name, _ext in INDEX_GRIDS.items():
    _T = math.prod(_ext)
    assert _name.startswith({True: "smem", False: "optin"}[_T <= 393216]) if _T <= 786432 else _name.startswith(("global", "decode64"))
    assert ("decode64" in _name) == (_T >= 2 ** 32) and ("T%32" not in _name or _name.endswith(f"={_T % 32}"))


def _grid_rows(g, ext, lo, P=20000):
    """P random rows inside [lo, lo + ext), plus the first and the last cell, shuffled"""
    cols = [lo[d] + torch.randint(0, ext[d], (P,), generator=g) for d in range(len(ext))]
    rows = torch.cat([torch.stack(cols, 1), torch.tensor([lo, [lo[d] + ext[d] - 1 for d in range(len(ext))]])])
    return rows[torch.randperm(rows.shape[0], generator=g)].contiguous()


@pytest.mark.parametrize("name", list(INDEX_GRIDS))
def test_unique_rows_grids(cuda, name):
    from sst_b200 import ops
    ext = INDEX_GRIDS[name]
    lo = [-3 * d - 2 for d in range(len(ext))]
    rows = _grid_rows(torch.Generator().manual_seed(len(name)), ext, lo)
    bounds = (lo, [lo[d] + ext[d] - 1 for d in range(len(ext))])
    ru, ri, rc = torch.unique(rows, dim=0, return_inverse=True, return_counts=True)
    for _ in range(2):
        gu, gi, gc = ops.unique_rows(rows.to(cuda), return_counts=True, bounds=bounds)
        assert torch.equal(gu.cpu(), ru) and torch.equal(gi.cpu(), ri) and torch.equal(gc.cpu(), rc)


@pytest.mark.parametrize("name", ["smem_k3", "optin_k3_T%32=31", "global_k3", "decode64_k3"])
def test_dynamic_scatter_grids(cuda, name):
    """dynamic scatter with coor_bounds that put the grid on each index path; rows on the first and the last cell and invalid rows"""
    from sst_b200 import ops
    ext = {"smem_k3": GRID, "global_k3": (9, 300, 400)}.get(name) or INDEX_GRIDS[name]
    g = torch.Generator().manual_seed(len(name) + 50)
    rows = _grid_rows(g, ext, [0, 0, 0])
    rows[torch.randperm(rows.shape[0], generator=g)[:40], torch.randint(0, 3, (40,), generator=g)] = -1
    coors = rows.to(torch.int32).contiguous()
    x = _randn(g, coors.shape[0], 4)
    bounds = ([0, 0, 0], [e - 1 for e in ext])
    for mode in ("max", "sum"):
        r_f, r_c, r_m, r_n = O.dynamic_point_to_voxel_forward(x.double(), coors, mode)
        for _ in range(2):
            g_f, g_c, g_m, g_n = ops.dynamic_point_to_voxel_forward(x.to(cuda), coors.to(cuda), mode, coor_bounds=bounds)
            assert torch.equal(g_c.cpu(), r_c) and torch.equal(g_m.cpu(), r_m) and torch.equal(g_n.cpu(), r_n)
            if mode == "max":
                assert torch.equal(g_f.cpu(), r_f.float())
            else:
                _assert_within(g_f, r_f, O.dynamic_point_to_voxel_forward(x.double().abs(), coors, "sum")[0], r_n.long(), mode)


def test_grid_beyond_2_34_is_refused(cuda):
    from sst_b200 import _lib as L, ops
    rows = torch.tensor([[0, 0], [5, 7]], device=cuda)
    with pytest.raises(L.SSTB200Error, match="error -3"):
        ops.unique_rows(rows, bounds=([0, 0], [2 ** 17, 2 ** 17 - 1]))
    co = torch.tensor([[0, 0, 0], [1, 2, 0]], dtype=torch.int32, device=cuda)
    with pytest.raises(L.SSTB200Error, match="error -3"):
        ops.dynamic_point_to_voxel_forward(torch.ones(2, 4, device=cuda), co, "max", coor_bounds=([0, 0, 0], [2 ** 17, 2 ** 17, 0]))
    with pytest.raises(L.SSTB200Error, match="error -3"):
        ops.get_inner_win_inds(torch.tensor([0, 2 ** 34], device=cuda))


def test_dynamic_scatter_drop_first_and_bounds(cuda):
    """the first sorted row is dropped: the (-1,-1,-1) row when a row has a negative coordinate, the smallest voxel otherwise; a
    non-negative row outside coor_bounds raises"""
    from sst_b200 import _lib as L, ops
    g = torch.Generator().manual_seed(8000)
    sizes = torch.randint(1, 9, (50,), generator=g).tolist()
    x = _randn(g, sum(sizes) + 3, 5)
    for invalid in (0, 3):
        coors = _voxel_coors(g, sizes, invalid)
        f = x[:coors.shape[0]].contiguous()
        _check_dynamic_scatter(ops, f.to(cuda), coors, f, "mean", cuda, 1, f"invalid={invalid}")
        _, vc, vm, _ = ops.dynamic_point_to_voxel_forward(f.to(cuda), coors.to(cuda), "mean")
        real = torch.unique(coors[(coors >= 0).all(1)], dim=0)
        assert torch.equal(vc.cpu(), real if invalid else real[1:])
        assert torch.equal(vm.cpu() < 0, (coors < 0).any(1) if invalid else (coors == real[0]).all(1))
    hi = coors.amax(0).tolist()
    with pytest.raises(L.SSTB200Error, match="outside coor_lo/hi"):
        ops.dynamic_point_to_voxel_forward(f.to(cuda), coors.to(cuda), "max", coor_bounds=([0, 0, 0], [hi[0], hi[1], hi[2] - 1]))


# ----------------------------------------------------------------------------------------------------------------------
# in-group ranks
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("max_id", [1000, 393215, 393216, 786431, 786432, 2 ** 21, 2 ** 32 + 5])
def test_ingroup_indices_grids(cuda, max_id):
    """groups of 1, 31, 32, 33 and random sizes; max_id + 1 = T on both sides of 393 216 and 786 432 cells, and past 2^32"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(max_id % 9973)
    sizes = [1, 31, 32, 33] + torch.randint(1, 70, (300,), generator=g).tolist()
    pool = torch.unique(torch.randint(1, max_id, (4 * len(sizes),), generator=g))
    ids = torch.cat([torch.tensor([0, max_id]), pool[torch.randperm(pool.numel(), generator=g)][:len(sizes) - 2]])
    grp = torch.repeat_interleave(ids, torch.tensor(sizes))
    grp = grp[torch.randperm(grp.numel(), generator=g)].contiguous()
    ref = O.ingroup_indices(grp)
    for _ in range(2):
        assert torch.equal(ops.get_inner_win_inds(grp.to(cuda)).cpu(), ref)


def test_ingroup_indices_one_large_group(cuda):
    """one group of 20 000 (the O(n^2 / 32) one-warp path) among small ones"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(8100)
    grp = torch.cat([torch.full((20000,), 7), torch.randint(0, 500, (3000,), generator=g)])
    grp = grp[torch.randperm(grp.numel(), generator=g)].contiguous()
    assert torch.equal(ops.get_inner_win_inds(grp.to(cuda)).cpu(), O.ingroup_indices(grp))


# ----------------------------------------------------------------------------------------------------------------------
# voxelisation
# ----------------------------------------------------------------------------------------------------------------------
def _face_points(g, vs, rng, n=30000):
    """points on voxel faces (lo + k vs formed in float32), one float32 step either side of them, at hi, just below lo, far outside,
    at -0.0, plus random points; every column picked independently"""
    cols = []
    for d in range(3):
        lo, hi, v = np.float32(rng[d]), np.float32(rng[3 + d]), np.float32(vs[d])
        k = np.arange(-2, int(np.ceil((hi - lo) / v)) + 3, dtype=np.float32)
        faces = (lo + k * v).astype(np.float32)
        cand = np.concatenate([faces, np.nextafter(faces, np.float32(np.inf)), np.nextafter(faces, np.float32(-np.inf)),
                               np.array([hi, np.nextafter(lo, np.float32(-np.inf)), lo, -0.0, 0.0, lo - 500, hi + 500],
                                        dtype=np.float32)])
        pick = torch.from_numpy(cand)[torch.randint(0, len(cand), (n,), generator=g)]
        rand = torch.rand(n, generator=g) * float(hi - lo + 4 * v) + float(lo - 2 * v)
        cols.append(torch.where(torch.rand(n, generator=g) < 0.8, pick, rand.float()))
    return torch.stack(cols, 1).contiguous()


@pytest.mark.parametrize("vs,rng", [((0.32, 0.32, 6.0), (-74.88, -74.88, -2.0, 74.88, 74.88, 4.0)),
                                    ((0.1, 0.1, 0.15), (0.0, -51.2, 0.0, 51.2, 51.2, 3.0))])
def test_voxelize_faces(cuda, vs, rng):
    """dynamic_voxelize (clamped) and voxelize_with_batch_idx (floor-divide, no clamp: negative offsets, -0.0) bit-exact"""
    from sst_b200 import ops
    from sst_b200.fsdv2_modules import voxelize_with_batch_idx
    g = torch.Generator().manual_seed(int(rng[3]))
    pts = _face_points(g, vs, rng)
    coors = torch.zeros((pts.shape[0], 3), dtype=torch.int32, device=cuda)
    ops.dynamic_voxelize(pts.to(cuda), coors, vs, rng, 3)
    assert torch.equal(coors.cpu(), O.dynamic_voxelize(pts, vs, rng))
    bidx = torch.randint(0, 4, (pts.shape[0],), generator=g)
    got = voxelize_with_batch_idx(pts.to(cuda), bidx.to(cuda), [float(np.float32(v)) for v in vs], list(rng))
    ref = O.voxelize_with_batch_idx(pts, bidx, [float(np.float32(v)) for v in vs], list(rng))
    assert (ref[:, 1:] < 0).any()
    assert torch.equal(got.cpu(), ref)


# ----------------------------------------------------------------------------------------------------------------------
# the reference's own CUDA voxel layer (oracle/_ref), when built
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_layer():
    try:
        m = build_ref.load_module()
    except Exception as e:  # e.g. a torch ABI mismatch
        pytest.skip(f"oracle/_ref not loadable: {e}")
    if m is None:
        pytest.skip("oracle/_ref/voxel_layer_ref.so not built")
    return m


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
@pytest.mark.parametrize("C", [3, 4, 36, 132, 300])
def test_dynamic_scatter_vs_reference_cuda(cuda, ref_layer, C, mode):
    """index outputs and max bit-exact; sum / mean within the reference's fp32 atomic accumulation (n 2^-24 sum|x| per element);
    backward bit-exact on the same forward outputs"""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(9000 + C)
    sizes = _edge_sizes(C, False) + torch.randint(1, 40, (100,), generator=g).tolist()
    coors = _voxel_coors(g, sizes, invalid=7).to(cuda)
    feats = _randn(g, coors.shape[0], C).to(cuda)
    r_f, r_c, r_m, r_n = ref_layer.dynamic_point_to_voxel_forward(feats, coors, mode)
    g_f, g_c, g_m, g_n = ops.dynamic_point_to_voxel_forward(feats, coors, mode)
    assert torch.equal(g_c, r_c) and torch.equal(g_m, r_m) and torch.equal(g_n, r_n)
    if mode == "max":
        assert torch.equal(g_f, r_f)
    else:
        a = O.dynamic_point_to_voxel_forward(feats.cpu().double().abs(), coors.cpu(), "sum")[0].to(cuda)
        n = g_n.double()[:, None]
        bound = 2.0 ** -22 * (g_f.double().abs() + (a if mode == "sum" else a / n) * n)
        assert ((g_f.double() - r_f.double()).abs() <= bound).all()
    grad = _randn(g, g_f.shape[0], C).to(cuda)
    r_g, g_g = torch.zeros_like(feats), torch.zeros_like(feats)
    ref_layer.dynamic_point_to_voxel_backward(r_g, grad, feats, g_f, g_m, g_n, mode)
    ops.dynamic_point_to_voxel_backward(g_g, grad, feats, g_f, g_m, g_n, mode)
    assert _same_bits(g_g, r_g)
