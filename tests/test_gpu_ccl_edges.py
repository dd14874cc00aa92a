"""GPU: FSD's instance grouping (csrc/ccl.cu, sstb200_connected_components) against the oracle at every distance, cell, grid, batch
and layout edge.

The call bins the centres into a uniform grid of cell dist * 1.01, tests each centre against the centres of its 3 x 3 cells with
the reference's fp32 arithmetic (sqrt(dx*dx + dy*dy) < dist, round-to-nearest at every step) and merges the edges in a lock-free
union-find.  Labels and the component count must be BIT-EXACT against oracle/fsd_oracle: the dense n x n form of the reference
(find_connected_components) up to DENSE_MAX centres, its k-d tree form (connected_components_large) above.

The cases put centre pairs exactly on the distance tie, one ulp either side of it and where fp32 and float64 disagree; centres on
cell boundaries, one ulp either side, on the far edge and outside the bounds on every side; grids of more than 2.5e5 cells per
axis, where fp32 binning put centres closer than dist two cells apart (the precondition re-emulates that binning in numpy, so the
case cannot lose its teeth), and grids on both sides of the 1e6-cells-per-axis refusal; one long chain in random index order, a
dyadic lattice whose fp32 distances are exact, many small components per warp; batches with empty samples, identical xy in
different samples and batch indices outside [0, B); n = 1, 255..257 and 65 537; strides 2, 3 and 7; degenerate bounds; dist = inf;
and NaN / +-inf centres with explicit and automatic bounds.

Every call runs after a "poison twin" (more centres, another dist, another grid) on the same context, writes into labels prefilled
with a sentinel that has GUARD words past n, and is made twice: once with the host count and once with the device count only.  The
guard words must keep the sentinel, both calls must give the same labels bit for bit, and the device count must equal the host one.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsd_oracle as FO

pytestmark = pytest.mark.gpu

SENTINEL = -7777
GUARD = 16
DENSE_MAX = 4096
f32 = np.float32


def _lib():
    from sst_b200 import _lib as L
    from sst_b200 import fsd_modules  # noqa: F401  (binds sstb200_connected_components)
    return L


def _call(c, pts, bidx, B, dist, lo, hi, host=True):
    """one sstb200_connected_components call; pts [n, stride] fp32 CUDA.  Returns (labels [n] CPU, device count, host count | None)"""
    L = _lib()
    n, stride = pts.shape
    buf = torch.full((n + GUARD,), SENTINEL, dtype=torch.int32, device=pts.device)
    num_dev = torch.full((1,), SENTINEL, dtype=torch.int32, device=pts.device)
    num_host = C.c_int32(SENTINEL)
    L.check(c, L.lib().sstb200_connected_components(c, pts.data_ptr(), stride, L.ptr(bidx), n, B, float(dist),
                                                    L.arr(C.c_float, [float(v) for v in lo]), L.arr(C.c_float, [float(v) for v in hi]),
                                                    buf.data_ptr(), num_dev.data_ptr(), C.byref(num_host) if host else None))
    buf = buf.cpu()
    assert torch.equal(buf[n:], torch.full((GUARD,), SENTINEL, dtype=torch.int32)), "a guard word past n was written"
    return buf[:n], int(num_dev.item()), (num_host.value if host else None)


def _poison(c, dev, n, dist):
    """a larger call with another dist and grid on the same context: the arena the real call carves is dirty"""
    g = torch.Generator().manual_seed(n)
    m = n + 777
    pts = ((torch.rand((m, 3), generator=g) - 0.5) * 60.0).to(dev)
    bidx = torch.randint(0, 3, (m,), generator=g, dtype=torch.int32).to(dev)
    d = 0.37 if not 0.3 < dist < 0.45 else 0.91
    _call(c, pts, bidx, 3, d, [-31.0, -29.0], [30.0, 33.0])


def _bounds(xy):
    return xy.amin(0).tolist(), xy.amax(0).tolist()


def oracle(pts, bidx, dist, B=None):
    """the reference's labels; centres whose batch index lies outside [0, B) get -1 (the call's contract)"""
    n = pts.shape[0]
    bidx = torch.zeros(n, dtype=torch.int32) if bidx is None else bidx
    B = int(bidx.max()) + 1 if B is None else B
    ok = (bidx >= 0) & (bidx < B)
    ref = torch.full((n,), -1, dtype=torch.int32)
    if ok.any():
        p, b = pts[ok], bidx[ok]
        dense = p.shape[0] <= DENSE_MAX or not torch.isfinite(p[:, :2]).all() or dist == float("inf")
        ref[ok] = (FO.find_connected_components(p, b, dist) if dense else FO.connected_components_large(p, b, dist)).int()
    return ref


def check(dev, pts, dist, bounds=None, bidx=None, B=None, ref=None):
    """pts [n, stride] fp32 CPU.  Both calls (host count, device count only) after a poison twin, against the oracle."""
    L = _lib()
    c = L.ctx(dev)
    n = pts.shape[0]
    if ref is None:
        ref = oracle(pts, bidx, dist, B)
    B = (1 if bidx is None else int(bidx.max()) + 1) if B is None else B
    lo, hi = bounds if bounds is not None else _bounds(pts[:, :2].double())
    p = pts.contiguous().to(dev)
    b = None if bidx is None else bidx.int().contiguous().to(dev)
    _poison(c, dev, n, dist)
    labels, num_dev, num_host = _call(c, p, b, B, dist, lo, hi, host=True)
    want = int(ref.max()) + 1 if n else 0
    assert num_host == want and num_dev == want, (num_host, num_dev, want)
    bad = torch.nonzero(labels != ref)[:, 0]
    assert bad.numel() == 0, f"{bad.numel()} of {n} labels differ, first at {bad[:5].tolist()}: {labels[bad[:5]].tolist()} vs {ref[bad[:5]].tolist()}"
    _poison(c, dev, n + 1, dist)
    again, num_dev2, _ = _call(c, p, b, B, dist, lo, hi, host=False)
    assert torch.equal(again, labels) and num_dev2 == want
    return labels


def d32(p, q):
    """the reference's fp32 distance of the rows of p and q (numpy float32: one rounding per operation)"""
    dx, dy = (p[:, 0] - q[:, 0]).astype(f32), (p[:, 1] - q[:, 1]).astype(f32)
    return np.sqrt((dx * dx + dy * dy).astype(f32)).astype(f32)


def d64(p, q):
    return np.sqrt((p[:, 0].astype(np.float64) - q[:, 0]) ** 2 + (p[:, 1].astype(np.float64) - q[:, 1]) ** 2)


def ulps(v, k):
    """v (fp32) moved k steps through the fp32 numbers (away from zero for k > 0 when v < 0)"""
    return (v.astype(f32).view(np.int32) + np.asarray(k, np.int32)).view(f32)


def _to_pts(xy, seed, extra=1):
    """centres [n, 2 + extra] in a random index order (the extra columns are z-like and never read)"""
    g = np.random.default_rng(seed)
    xy = xy[g.permutation(xy.shape[0])]
    return torch.from_numpy(np.concatenate([xy, g.random((xy.shape[0], extra), dtype=f32)], 1).astype(f32))


# ---- distance ties ------------------------------------------------------------------------------------------------------------
def _tie_pairs(seed, dist, n):
    """n pairs (p, q) whose fp32 distance is exactly dist, on a grid centred at the origin (fine ulps) and spaced 5 dist apart, so
    that no two pairs interact"""
    g = np.random.default_rng(seed)
    k = int(np.ceil(np.sqrt(n * 1.5)))
    gx, gy = np.meshgrid(np.arange(k) - k // 2, np.arange(k) - k // 2)
    base = np.stack([gx.ravel(), gy.ravel()], 1)
    p = (base * 5.0 * dist + g.random(base.shape) * dist).astype(f32)
    th = g.random(p.shape[0]) * 2 * np.pi
    q0 = (p + dist * np.stack([np.cos(th), np.sin(th)], 1)).astype(f32)
    q, found = q0.copy(), np.zeros(p.shape[0], bool)
    for kx in range(-24, 25):
        for ky in range(-24, 25):
            cand = np.stack([ulps(q0[:, 0], kx), ulps(q0[:, 1], ky)], 1)
            hit = (d32(p, cand) == f32(dist)) & ~found
            q[hit], found = cand[hit], found | hit
    assert found.sum() >= n, (found.sum(), n)
    return p[found][:n], q[found][:n]


@pytest.mark.parametrize("dist", [0.5, 0.6, 0.3])
def test_distance_ties(cuda, dist):
    """pairs at fp32 distance == dist (no edge: the test is strict), the same pairs one ulp inward and outward, and pairs where the
    fp32 and float64 decisions disagree: the call follows fp32, like the reference"""
    dist = float(f32(dist))
    n = 150
    p, q = _tie_pairs(7, dist, 3 * n)
    qq = q.copy()  # q.x one ulp toward p, or one ulp away from it
    qq[n:2 * n, 0] = np.nextafter(q[n:2 * n, 0], p[n:2 * n, 0])
    qq[2 * n:, 0] = np.nextafter(q[2 * n:, 0], np.where(q[2 * n:, 0] > p[2 * n:, 0], f32(np.inf), f32(-np.inf)))
    dd, dd64 = d32(p, qq), d64(p, qq)
    edge32, edge64 = dd < f32(dist), dd64 < dist
    assert (dd[:n] == f32(dist)).all() and not edge32[:n].any()
    assert edge32[n:2 * n].sum() >= n // 4 and not edge32[2 * n:].any()
    assert (edge32 != edge64).sum() >= 10, "the case needs pairs where fp32 and float64 decide differently"
    pts = _to_pts(np.concatenate([p, qq]), 1)
    labels = check(cuda, pts, dist)
    assert int(labels.max()) + 1 == 2 * 3 * n - int(edge32.sum())
    # and with a dyadic dist, axis-aligned pairs whose fp32 differences are exact
    x = (np.arange(200, dtype=f32) * 4 + 3).astype(f32)
    p2 = np.stack([x, np.full_like(x, 5.0)], 1)
    q2 = p2 + np.array([0.5, 0.0], f32)
    q2[100:150, 0] = ulps(q2[100:150, 0], -1)
    q2[150:, 0] = ulps(q2[150:, 0], 1)
    check(cuda, _to_pts(np.concatenate([p2, q2]).astype(f32), 2), 0.5)


# ---- cell boundaries ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dist", [0.6, 0.25])
def test_cell_boundaries(cuda, dist):
    """centres at x0 + k cell, one ulp either side and at the far edge x0 + nx cell (k every 4th boundary, so that the clusters
    stay apart), the same in y, and centres outside the bounds on all four sides within dist of in-range ones (clamped into the
    border cells), far outside, and far outside beside an in-range centre of the same border cell"""
    d = float(f32(dist))
    cell = d * 1.01
    lo = np.array([-3.3, 1.7], f32)
    span = 30.5 * cell
    hi = (lo + f32(span)).astype(f32)
    nx = int((float(hi[0]) - float(lo[0])) / cell) + 1
    assert nx == 31
    rows = []

    def cluster(axis, k, other):
        b = f32(float(lo[axis]) + k * cell)
        vals = [ulps(np.array([b]), -1)[0], b, ulps(np.array([b]), 1)[0], f32(b - f32(0.999 * d)), f32(b + f32(0.999 * d))]
        for v in vals:
            rows.append((v, other) if axis == 0 else (other, v))

    for k in list(range(0, 29, 4)) + [nx]:
        cluster(0, k, f32(lo[1] + 26.5 * cell))
    for k in range(0, 17, 4):
        cluster(1, k, f32(lo[0] + 2.5 * cell))
    ym, ym2, xm = f32(lo[1] + 8.5 * cell), f32(lo[1] + 12.5 * cell), f32(lo[0] + 14.5 * cell)
    rows += [(lo[0] - f32(0.5 * d), ym), (lo[0] + f32(0.45 * d), ym),          # left
             (hi[0] + f32(0.5 * d), ym2), (hi[0] - f32(0.45 * d), ym2),        # right
             (xm, lo[1] - f32(0.5 * d)), (xm, lo[1] + f32(0.45 * d)),          # bottom
             (xm, hi[1] + f32(0.5 * d)), (xm, hi[1] - f32(0.45 * d)),          # top
             (lo[0] - 100, lo[1] - 100), (lo[0] - 100 + f32(0.9 * d), lo[1] - 100),   # far outside, one border cell, connected
             (hi[0] + 1e4, hi[1] + 50), (hi[0] + 1e4, hi[1] + 50 + f32(0.9 * d)),
             (lo[0] - 100, f32(lo[1] + 20.5 * cell)), (lo[0] + f32(0.1 * d), f32(lo[1] + 20.5 * cell))]  # same cell, far apart
    xy = np.array(rows, dtype=f32)
    pts = _to_pts(xy, 3)
    ref = oracle(pts, None, d)
    assert int(ref.max()) + 1 == 8 + 1 + 5 + 4 + 2 + 2, "every cluster and every outside pair is one component"
    check(cuda, pts, d, bounds=(lo.tolist(), hi.tolist()), ref=ref)
    check(cuda, pts, d, ref=ref)  # bounds over all centres: nothing clamped


# ---- large grids ----------------------------------------------------------------------------------------------------------------
def _old_fp32_cells(v, v0, dist):
    """the binning before fp64: floorf((v - x0) * (1 / (dist * 1.01f))) in fp32"""
    cell = f32(f32(dist) * f32(1.01))
    inv = f32(f32(1.0) / cell)
    return np.floor(((v.astype(f32) - f32(v0)).astype(f32) * inv).astype(f32)).astype(np.int64)


def _new_cells(v, v0, dist):
    return np.floor((v.astype(np.float64) - np.float64(f32(v0))) / (np.float64(f32(dist)) * 1.01)).astype(np.int64)


@pytest.mark.parametrize("dist", [6e-4, 3e-4])
def test_large_grid_binning(cuda, dist):
    """a thin strip, x in [-80, 80] (264 027 and 528 053 cells), y a few cells: pairs at 0.97..1.0 dist.  Binned in fp32, some of
    these pairs land two cells apart and the 3 x 3 search never compares them (asserted by emulation below, together with the
    labels that binning would give); binned in fp64 none do."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree
    d = float(f32(dist))
    cell = d * 1.01
    lo, hi = [-80.0, 0.0], [80.0, float(f32(3 * cell))]
    g = np.random.default_rng(11)
    m = 60000  # a quarter over the whole strip, the rest at x > 20 where fp32 binning errs most; mostly along x
    ax = np.where(g.random(m) < 0.25, g.uniform(-80, 80, m), g.uniform(20, 80, m))
    a = np.stack([ax, g.uniform(0, 3 * cell, m)], 1).astype(f32)
    th = g.normal(0, 0.05, m) + np.pi * (g.random(m) < 0.5)
    r = g.uniform(0.97, 1.0, m) * d
    b = (a + r[:, None] * np.stack([np.cos(th), np.sin(th)], 1)).astype(f32)
    xy = np.concatenate([a, b])
    pts = _to_pts(xy, 5)
    xy = pts[:, :2].numpy()
    # every pair the reference connects, and where each binning puts its ends
    pairs = cKDTree(xy.astype(np.float64)).query_pairs(d * 1.001 + 1e-6, output_type="ndarray")
    pairs = pairs[d32(xy[pairs[:, 0]], xy[pairs[:, 1]]) < f32(d)]
    old = [np.abs(_old_fp32_cells(xy[pairs[:, 0], ax], lo[ax], d) - _old_fp32_cells(xy[pairs[:, 1], ax], lo[ax], d)) for ax in (0, 1)]
    new = [np.abs(_new_cells(xy[pairs[:, 0], ax], lo[ax], d) - _new_cells(xy[pairs[:, 1], ax], lo[ax], d)) for ax in (0, 1)]
    missed = (old[0] > 1) | (old[1] > 1)
    assert missed.sum() >= 10, f"only {missed.sum()} connected pairs fall two cells apart under fp32 binning"
    assert ((new[0] <= 1) & (new[1] <= 1)).all()
    ref = oracle(pts, None, d)
    n = xy.shape[0]
    kept = pairs[~missed]
    gr = coo_matrix((np.ones(kept.shape[0], bool), (kept[:, 0], kept[:, 1])), shape=(n, n))
    old_labels = torch.from_numpy(connected_components(gr, directed=False)[1]).int()
    assert not torch.equal(old_labels, ref), "fp32 binning would still give the reference's labels"
    check(cuda, pts, d, bounds=(lo, hi), ref=ref)


def test_grid_size_limit(cuda):
    """a grid just under 1e6 cells per axis is labelled (pairs at 0.98 dist up to its far end), one just over it is refused on
    either axis"""
    L = _lib()
    d = float(f32(1e-3))
    cell = d * 1.01
    under, over = float(f32(999_999.5 * cell)), float(f32(1_000_000.5 * cell))
    assert under / cell <= 1e6 < over / cell
    g = np.random.default_rng(13)
    m = 3000
    a = np.stack([np.concatenate([g.uniform(0, under, m - 200), under - g.uniform(0, 0.05, 200)]), np.zeros(m)], 1).astype(f32)
    b = (a + np.array([0.98 * d, 0.0])).astype(f32)
    pts = _to_pts(np.concatenate([a, b]), 6)
    ref = check(cuda, pts, d, bounds=([0.0, 0.0], [under, 0.0]))
    assert int(ref.max()) + 1 < pts.shape[0]
    c = L.ctx(cuda)
    p = pts.to(cuda)
    for hi in ([over, 0.0], [0.0, over]):
        with pytest.raises(L.SSTB200Error):
            _call(c, p, None, 1, d, [0.0, 0.0], hi)


# ---- union-find stress ----------------------------------------------------------------------------------------------------------
def test_long_chain_random_order(cuda):
    """80 000 centres 0.9 dist apart along a wavy line over ~71 000 cells, in random index order (unions arrive in adversarial
    order), with five links widened to 1.1 dist: six components"""
    d = 0.01
    n = 80000
    g = np.random.default_rng(17)
    gaps = np.full(n - 1, 0.9 * d)
    cut = g.choice(n - 1, 5, replace=False)
    gaps[cut] = 1.1 * d
    x = np.concatenate([[0.0], np.cumsum(gaps)]) - 300.0
    y = 0.002 * np.sin(np.arange(n) * 0.01)
    pts = _to_pts(np.stack([x, y], 1).astype(f32), 7)
    ref = oracle(pts, None, d)
    assert int(ref.max()) + 1 == 6
    check(cuda, pts, d)


def test_dyadic_lattice(cuda):
    """a 48 x 48 lattice of spacing 0.5 near the origin: every fp32 distance is exact, so dist 0.5 gives no edge and dist one ulp
    above 0.5 gives one component"""
    i, j = np.meshgrid(np.arange(48), np.arange(48))
    xy = (np.stack([i.ravel(), j.ravel()], 1) * 0.5 - 3.0).astype(f32)
    pts = _to_pts(xy, 8)
    labels = check(cuda, pts, 0.5)
    assert int(labels.max()) + 1 == xy.shape[0]
    up = float(np.nextafter(f32(0.5), f32(1.0)))
    labels = check(cuda, pts, up)
    assert int(labels.max()) == 0


@pytest.mark.parametrize("shuffle", [False, True])
def test_many_small_components(cuda, shuffle):
    """20 000 components of 1..4 centres each, members at consecutive indices (many components per warp) or shuffled"""
    d = 0.2
    g = np.random.default_rng(19)
    sizes = g.integers(1, 5, 20000)
    rows = []
    for k, s in enumerate(sizes):
        c = np.array([(k % 200) * 1.0, (k // 200) * 1.0])
        for t in range(s):
            rows.append(c + np.array([0.15 * t, 0.0]))
    xy = np.array(rows, dtype=f32)
    pts = _to_pts(xy, 9) if shuffle else torch.from_numpy(np.concatenate([xy, np.zeros((xy.shape[0], 1), f32)], 1))
    labels = check(cuda, pts, d)
    assert int(labels.max()) + 1 == sizes.size


# ---- batches ----------------------------------------------------------------------------------------------------------------------
def _batch(seed, occupied, per):
    g = torch.Generator().manual_seed(seed)
    xs, bs = [], []
    for b in occupied:
        p, _ = FO.synth_centres(seed + b, 1, per, spread=8.0, blob=0.3, blobs=20)
        xs.append(p)
        bs.append(torch.full((per,), b, dtype=torch.int32))
    pts, bidx = torch.cat(xs), torch.cat(bs)
    if 2 in occupied and 3 in occupied:  # identical xy in samples 2 and 3: never connected to each other
        pts[bidx == 3, :2] = pts[bidx == 2, :2]
    perm = torch.randperm(pts.shape[0], generator=g)
    return pts[perm].contiguous(), bidx[perm].contiguous()


def test_batches(cuda):
    """B = 16 with empty samples between occupied ones, indices interleaved, identical xy in samples 2 and 3"""
    occupied = [0, 2, 3, 7, 8, 15]
    pts, bidx = _batch(23, occupied, 500)
    labels = check(cuda, pts, 0.6, bidx=bidx, B=16)
    l2, l3 = labels[bidx == 2], labels[bidx == 3]
    assert int(l2.max()) < int(l3.min())
    # a trailing run of empty samples
    sub = bidx < 8
    check(cuda, pts[sub].contiguous(), 0.6, bidx=bidx[sub].contiguous(), B=16)


def test_batch_index_out_of_range(cuda):
    """batch indices -1 and B: refused when the host count is requested; with the device count only, labelled -1 and the rest as
    the reference labels the valid centres"""
    L = _lib()
    pts, bidx = _batch(29, [0, 1, 3], 400)
    bidx = bidx.clone()
    bidx[::37] = 4
    bidx[5::41] = -1
    ref = oracle(pts, bidx, 0.6, B=4)
    assert int((ref == -1).sum()) == int(((bidx < 0) | (bidx >= 4)).sum()) > 0
    c = L.ctx(cuda)
    p, b = pts.to(cuda), bidx.to(cuda)
    _poison(c, cuda, pts.shape[0], 0.6)
    with pytest.raises(L.SSTB200Error):
        _call(c, p, b, 4, 0.6, *_bounds(pts[:, :2].double()), host=True)
    _poison(c, cuda, pts.shape[0], 0.6)
    labels, num_dev, _ = _call(c, p, b, 4, 0.6, *_bounds(pts[:, :2].double()), host=False)
    assert torch.equal(labels, ref) and num_dev == int(ref.max()) + 1


# ---- sizes and layouts ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 255, 256, 257, 65537])
def test_sizes(cuda, n):
    p, _ = FO.synth_centres(31 + n, 1, n, spread=10.0 + n / 200, blob=0.3, blobs=max(1, n // 40))
    check(cuda, p, 0.4)


@pytest.mark.parametrize("stride", [2, 3, 7])
def test_strides(cuda, stride):
    """columns past x, y hold NaN: never read"""
    p, b = FO.synth_centres(37, 2, 1500, spread=10.0, blob=0.3, blobs=40)
    pts = torch.full((p.shape[0], stride), float("nan"))
    pts[:, :2] = p[:, :2]
    ref = oracle(p, b, 0.5)
    check(cuda, pts, 0.5, bidx=b, ref=ref)


def test_degenerate_bounds_and_infinite_dist(cuda):
    """xy_max == xy_min (every centre in one cell, clamped) and dist = inf (one component per sample)"""
    p, b = FO.synth_centres(41, 3, 700, spread=6.0, blob=0.3, blobs=30)
    check(cuda, p, 0.5, bidx=b, bounds=([1.0, -2.0], [1.0, -2.0]))
    same = torch.zeros((300, 3))
    same[:, :2] = torch.tensor([4.25, -1.5])
    check(cuda, same, 0.5)
    labels = check(cuda, p, float("inf"), bidx=b)
    assert torch.equal(labels, b.int())


# ---- non-finite centres -----------------------------------------------------------------------------------------------------------
def _nonfinite(seed):
    p, b = FO.synth_centres(seed, 2, 800, spread=10.0, blob=0.3, blobs=30)
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(p.shape[0], generator=g)[:60]
    vals = [float("nan"), float("inf"), float("-inf")]
    for k, i in enumerate(idx.tolist()):
        p[i, k % 2] = vals[k % 3]
        if k % 5 == 0:
            p[i, 1 - k % 2] = vals[(k + 1) % 3]
    return p, b, idx


def test_nonfinite_centres_explicit_bounds(cuda):
    """NaN, +inf and -inf in x or y: singletons, numbered in index order like the reference"""
    p, b, idx = _nonfinite(43)
    for dist in (0.5, float("inf")):
        labels = check(cuda, p, dist, bidx=b, bounds=([-12.0, -12.0], [12.0, 12.0]))
        lab = labels[idx]
        assert all(int((labels == v).sum()) == 1 for v in lab.tolist())


def test_nonfinite_centres_automatic_bounds(cuda):
    """the wrapper's automatic bounds span the finite centres only: the same labels as the reference, also when no centre is
    finite"""
    from sst_b200 import fsd_modules as FM
    L = _lib()
    c = L.ctx(cuda)
    p, b, _ = _nonfinite(47)
    for dist in (0.5, float("inf")):
        ref = oracle(p, b, dist)
        _poison(c, cuda, p.shape[0], dist)
        labels, num = FM.connected_components(p.to(cuda), b.to(cuda), dist)
        assert num == int(ref.max()) + 1 and torch.equal(labels.cpu(), ref)
    bad = torch.tensor([[float("nan"), 1.0, 0.0], [float("inf"), float("-inf"), 0.0], [2.0, float("nan"), 0.0]])
    ref = oracle(bad, None, 0.5)
    assert torch.equal(ref, torch.arange(3, dtype=torch.int32))
    _poison(c, cuda, 3, 0.5)
    labels, num = FM.connected_components(bad.to(cuda), None, 0.5)
    assert num == 3 and torch.equal(labels.cpu(), ref)
