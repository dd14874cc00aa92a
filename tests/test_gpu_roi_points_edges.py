"""GPU: points-in-boxes (csrc/roiaware.cu: sstb200_points_in_boxes), RoIAwarePool3d (sstb200_roiaware_pool3d_plan / _forward /
_backward) and FSD's RoI point pooling (csrc/roi_pool.cu: sstb200_dynamic_point_pool, plain and mixed) against the fp32 oracles
(oracle/roiaware_oracle.py, oracle/roi_pool_oracle.py) and a float64 restatement, through the C ABI, at every place the kernels change
route.  Each case asserts that the layout it is named for actually happened, from the constants read out of the sources.

points_in_boxes, first mode: boxes are staged PIB_CHUNK (256) at a time and a block stops once every live thread has a hit
(__syncthreads_and).  T = 0, 1, 255, 256, 257, 512, 513 with B = 1, 3, 7 and M = 1, 255, 256, 257, 513; a point's only box sits in
chunk 0, 1 and the last chunk, and a point inside boxes of several chunks must get the lowest index across the chunk boundary; a block
whose 255 threads hit in chunk 0 while one thread hits only in the last chunk.
points_in_boxes, all mode: a tile of min(64, PIB_BITS_SMEM / row bytes) rows writes its contiguous output as a scalar head up to
16-byte alignment, an int4 body and a scalar tail.  T = 1, 3, 5, 31, 32, 33, 257 (every head length, body and tail), T = 12288, 12289
and 20000 (rows per block 64, 63, 39), M not a multiple of the rows, and `out` at byte offsets 0, 4, 8 and 12.  The head is taken from
the address; a CPU emulation shows that the element-index head the kernel used before puts the int4 body off its 16-byte alignment
for every offset but 0.  T = 786432 (one row per block) runs; T = 786433 is refused with SSTB_ERR_UNSUPPORTED.
The BEV grid (box3d.cuh), through both RoIAwarePool3d and dynamic_point_pool: the table (grid_table_size) at N = 512 | 513 (1024 ->
2048 buckets) and at N = 2^23 + 1 (capped at 2^24); a 40 m x 40 m RoI over 512 points takes the footprint fallback (more cells than
buckets) and the same RoI over more points the hashed route, with the same pairs; RoIs and points at |x|, |y| = 1e4, 3.3e4 (past the
32767-cell clamp) and 1e5 m, at 0, 45 deg and one fp32 step off 45 deg, with points a few fp32 steps either side of every corner of
the box and on integer cell boundaries; NaN x / y (never admitted; a NaN z is admitted when x, y are inside, as the reference's
|z - cz| > h / 2 test does); (cell, batch) triples found on the CPU to share a bucket, across cells and across batches, and one cell under batch ids 0 and the
table size (same bucket, same cell key: only the batch test keeps them apart); negative dims.
RoIAwarePool3d: nvox = 1, 63, 64, 65, 255, 256 and 255 (1 x 1 x 255), (255, 255, 255) plan-only, C = 1, 31, 32, 33, 64, 65, 257,
occupied slots on both sides of the pool kernel's 32-slot warp edges with empty warps between, m = 1 (nothing kept), 2 and a crowded
voxel whose m - 1 lowest point indices must be kept, points on the top face and under the bottom (the clamped voxel index), max with
ties, NaN and -inf, batch ids with empty samples; the backward at N = 255, 256, 65535, 65536 (the pad key N and the sort's
bits_for(N + 1)), with most pairs not kept, and with one point held by 50 overlapping RoIs; a pair key of exactly 64 bits is planned,
65 is refused.
dynamic_point_pool: n_pts = 256, 257, 65536, 65537, 2^24, 2^24 + 1 (1 to 4 radix-select passes), each with a RoI whose hits exceed
take and whose indices share their low bytes and differ only in the top digit; take = 1, 2, 255, 256, 257, 4095, 4096, 4097, 8191,
8192 (8193 refused); max_all_pts mid-RoI, on a RoI boundary, on the last pair and one short of it, per call and per sample; fake rows
for empty samples first, in the middle and last; unsorted per-sample RoIs and negative batch ids refused; the mixed form against
per-sample calls.

Contracts.  Membership (points_in_boxes, RoIAwarePool3d's kept points, dynamic_point_pool's indices) is bit-exact against the fp32
oracles (with cos / sin of the fp32 angle taken from the device, as the kernels take them: the correctly rounded values can differ by
an ulp, which decides points a few fp32 steps from a corner near the origin), and against the float64 in-box test for every (box, point) farther than delta from every face, delta bounding the fp32
arithmetic: u (|rz + pi/2| + 12) (|dx| + |dy|) + 4 u (|z| + |cz| + l + w + h), u = 2^-24.  RoIAwarePool3d's forward is bitwise
(argmax included) and avg is within count u sum|x| of the float64 mean; the backward is bitwise against a numpy emulation of the
kernel's sequential fp32 sum in (roi, voxel) order, within (k + 2) u sum|terms| of float64 (k terms; the 2 covers the rounded 1 / count
and product), and bit-identical from run to run.  dynamic_point_pool's idx, roi and is_in_margin are exact and raw xyz bitwise; local
xyz and boundary offsets are within the error of the kernel's fp32 rotation of the centre offset (the bound above on |dx| + |dy|,
2 u (|cz| + |lz|) for z, and the rounding of half-dims plus offset), not a fixed tolerance.  Every output is pre-filled with a sentinel
(a NaN payload no arithmetic makes, or 0x5A5A5A5A for integers, since 0xFF bytes read as the valid -1) and has guard space past its
end; every element that must be written is, and nothing past the end is.  Every pooling case runs right after a larger call on the
same context, so the arena it reuses is dirty.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import roi_pool_oracle as RO, roiaware_oracle as RA

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
GUARD = 64
ISENT = 0x5A5A5A5A        # integer sentinel: no index, count or flag takes this value
FSENT = 0x7FA5A5A5        # float sentinel: a NaN payload that no arithmetic produces
ERR_ARG, ERR_UNSUPPORTED = -2, -3
EXTRA = [0.5, 0.5, 0.5]


def _src(name):
    return open(os.path.join(ROOT, "sst_b200", "csrc", name)).read()


def _define(src, name):
    return int(eval(re.search(rf"#define {name} ([0-9 ()*]+)", src).group(1), {"__builtins__": {}}))


RA_SRC, RP_SRC, GRID_SRC = _src("roiaware.cu"), _src("roi_pool.cu"), _src("box3d.cuh")
PIB_THREADS, PIB_CHUNK = _define(RA_SRC, "PIB_THREADS"), _define(RA_SRC, "PIB_CHUNK")
PIB_MAX_ROWS, PIB_BITS_SMEM = _define(RA_SRC, "PIB_MAX_ROWS"), _define(RA_SRC, "PIB_BITS_SMEM")
RP_MAX_INBOX = _define(RP_SRC, "RP_MAX_INBOX")
CELL_CLAMP = _define(GRID_SRC, "RP_CELL_CLAMP")
HASH = tuple(int(v) for v in re.search(r"\(uint32_t\)cx \* (\d+)u \^ \(uint32_t\)cy \* (\d+)u \^ \(uint32_t\)b \* (\d+)u", GRID_SRC).groups())
assert "uint32_t T = 1024;" in GRID_SRC and "T < 2u * (uint32_t)num_pts && T < (1u << 24)" in GRID_SRC
assert "nc > (long long)g.mask + 1" in GRID_SRC


def _box_test_dev(pts, boxes):
    """roi_pool_oracle.box_test with cos / sin of the fp32 angle taken from the device (cosf / sinf, as the kernels and the reference's
    kernel take them) instead of correctly rounded: the two can differ by an ulp, which decides points a few fp32 steps from a corner"""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    cx, cy, zb, w, l, h, rz = boxes.unbind(1)
    cz = (zb.double() + h.double() / 2).float()
    ang = (rz.double() + math.pi / 2).float()
    ca, sa = torch.cos(ang.cuda()).cpu(), torch.sin(ang.cuda()).cpu()
    sx, sy = x[None] - cx[:, None], y[None] - cy[:, None]
    lx = (sx.double() * ca.double()[:, None] - (sy * sa[:, None]).double()).float()
    ly = (sy.double() * ca.double()[:, None] + (sx * sa[:, None]).double()).float()
    inside = ~((z[None] - cz[:, None]).abs() > (h / 2)[:, None])
    inside &= (lx > -(l / 2)[:, None]) & (lx < (l / 2)[:, None]) & (ly > -(w / 2)[:, None]) & (ly < (w / 2)[:, None])
    return inside, lx, ly, cz


@pytest.fixture(autouse=True)
def _device_trig(monkeypatch):
    monkeypatch.setattr(RO, "box_test", _box_test_dev)
    monkeypatch.setattr(RA, "box_test", _box_test_dev)


def _L():
    from sst_b200 import _lib as L, ops  # noqa: F401  (ops binds the entry points)
    return L


def _bits(t):
    """fp32 as bit patterns (-0.0 != 0.0), every NaN as one pattern: NaN payloads differ between CPU and GPU arithmetic"""
    t = t.cpu().contiguous()
    return torch.where(torch.isnan(t), torch.full_like(t, float("nan")), t).view(torch.int32)


# ---- Python mirrors of the kernels' layout decisions ---------------------------------------------------------------------------
def table_size(n):
    t = 1024
    while t < 2 * n and t < (1 << 24):
        t <<= 1
    return t


def pib_rows(T):
    return min(PIB_MAX_ROWS, PIB_BITS_SMEM // (((T + 31) // 32) * 4))


def radix_passes(n):
    return (max((n - 1).bit_length(), 1) + 7) // 8


def bits_for(n):
    return max(n - 1, 0).bit_length()


def bucket(cx, cy, b, mask):
    m = 0xFFFFFFFF
    return ((((cx & m) * HASH[0]) & m) ^ (((cy & m) * HASH[1]) & m) ^ (((b & m) * HASH[2]) & m)) & mask


def cell(v):
    f = np.floor(np.float32(v))
    if not f >= -CELL_CLAMP:
        return -CELL_CLAMP
    return CELL_CLAMP if f > CELL_CLAMP else int(f)


def footprint_cells(roi, extra):
    """cells under the axis-aligned footprint of the enlarged RoI, as for_each_hit computes them (fp32)"""
    f = np.float32
    cx, cy, _, w, l, _, rz = (f(v) for v in roi)
    w, l = f(w + f(extra[0])), f(l + f(extra[1]))
    ang = f(float(rz) + math.pi / 2)
    ca, sa = abs(f(math.cos(ang))), abs(f(math.sin(ang)))
    hl, hw = f(0.5) * l, f(0.5) * w
    pad = f(0.01) + f(1e-6) * (abs(cx) + abs(cy))
    rx, ry = ca * hl + sa * hw + pad, sa * hl + ca * hw + pad
    nx, ny = cell(cx + rx) - cell(cx - rx) + 1, cell(cy + ry) - cell(cy - ry) + 1
    return max(nx, 0) * max(ny, 0)


# ---- float64 references ----------------------------------------------------------------------------------------------------------
def _local64(p, b):
    """float64 local frame of points p [..., 3] in boxes b [..., 7] (broadcast): lx, ly, dz from the centre, the error scale of the
    kernel's fp32 rotation (u (|ang| + 12)(|dx| + |dy|)) and of its z (2 u (|cz| + |dz|))"""
    ang = b[..., 6] + math.pi / 2
    sx, sy = p[..., 0] - b[..., 0], p[..., 1] - b[..., 1]
    ca, sa = torch.cos(ang), torch.sin(ang)
    lx, ly = sx * ca - sy * sa, sx * sa + sy * ca
    cz = b[..., 2] + b[..., 5] / 2
    dz = p[..., 2] - cz
    return lx, ly, dz, U * (ang.abs() + 12) * (sx.abs() + sy.abs()), 2 * U * (cz.abs() + dz.abs())


def inbox64(pts, boxes, chunk=64):
    """float64 in-box test of every (box, point) [T, M] and the pairs within delta of a face (left to the fp32 comparison)"""
    ins, nears = [], []
    p = pts.double()[None]
    for k0 in range(0, boxes.shape[0], chunk):
        b = boxes[k0:k0 + chunk].double()[:, None]
        lx, ly, dz, exy, ez = _local64(p, b)
        hl, hw, hh = b[..., 4] / 2, b[..., 3] / 2, b[..., 5] / 2
        inside = (lx.abs() < hl) & (ly.abs() < hw) & ~(dz.abs() > hh)
        delta = exy + ez + 4 * U * (p[..., 2].abs() + b[..., 3].abs() + b[..., 4].abs() + b[..., 5].abs())
        near = ((hl - lx.abs()).abs() <= delta) | ((hw - ly.abs()).abs() <= delta) | ((hh - dz.abs()).abs() <= delta)
        ins.append(inside), nears.append(near)
    if not ins:
        z = torch.zeros((0, pts.shape[0]), dtype=torch.bool)
        return z, z
    return torch.cat(ins), torch.cat(nears)


def check_inside(inside, pts, boxes):
    """inside [T, M] from a kernel: bit-exact against the fp32 oracle, and against float64 off the faces; returns the clear pairs"""
    assert torch.equal(inside, RA.membership(pts, boxes)[0])
    in64, near = inbox64(pts, boxes)
    clear = ~near
    bad = (inside != in64) & clear
    assert not bad.any(), f"{int(bad.sum())} pairs farther than delta from every face disagree with float64, first {bad.nonzero()[:4].tolist()}"
    return int(clear.sum())


# ---- points_in_boxes through the C ABI ---------------------------------------------------------------------------------------------
def pib_abi(c, pts, boxes, mode, offset=0):
    """out at `offset` int32 elements into a sentinel-filled buffer with GUARD elements past its end"""
    L = _L()
    B, M, _ = pts.shape
    T = boxes.shape[1]
    n = B * M * (T if mode == 1 else 1)
    buf = torch.full((offset + n + GUARD,), ISENT, dtype=torch.int32, device="cuda")
    p, b = pts.float().contiguous().cuda(), boxes.float().contiguous().cuda()
    rc = L.lib().sstb200_points_in_boxes(c, p.data_ptr(), b.data_ptr(), B, M, T, mode, buf.data_ptr() + 4 * offset)
    assert rc == 0, L.lib().sstb200_last_error(c)
    buf = buf.cpu()
    assert (buf[:offset] == ISENT).all() and (buf[offset + n:] == ISENT).all(), "an int32 outside the output was written"
    out = buf[offset:offset + n]
    assert (out != ISENT).all(), "an output element was not written"
    return out.view(B, M, T) if mode == 1 else out.view(B, M)


def _pib_boxes(T, slots, pattern):
    """decoys far from every point, and at slots[j] a box over x in (j - 0.4, j + 0.4) (pattern 0: a point at x = j is in that box
    only) or over x in (-0.5, j + 0.5) (pattern 1: it is in boxes slots[j:], across chunks, and the lowest must win)"""
    k = torch.arange(T, dtype=torch.float32)
    boxes = torch.stack([1000.0 + 3.0 * k, torch.full_like(k, 50.0), torch.full_like(k, -1.0), torch.ones_like(k), torch.ones_like(k),
                         torch.full_like(k, 2.0), torch.zeros_like(k)], 1)
    for j, s in enumerate(slots):
        a, b = (j - 0.4, j + 0.4) if pattern == 0 else (-0.5, j + 0.5)
        boxes[s] = torch.tensor([(a + b) / 2, 0.0, -1.0, b - a, 2.0, 2.0, 0.0])   # yaw 0: w spans x, l spans y
    return boxes


def _pib_points(M, nslot, seed):
    """point i at x = j + noise, j = i mod (nslot + 1); j = nslot is in no box"""
    g = torch.Generator().manual_seed(seed)
    j = torch.arange(M) % (nslot + 1)
    x = j.float() + (torch.rand(M, generator=g) - 0.5) * 0.6
    x[j == nslot] += 1.5
    return torch.stack([x, (torch.rand(M, generator=g) - 0.5) * 1.6, (torch.rand(M, generator=g) - 0.5) * 1.8], 1), j


@pytest.mark.parametrize("T", [0, 1, 255, 256, 257, 512, 513])
def test_pib_first_chunks(cuda, T):
    """the lowest containing box across PIB_CHUNK-box chunks, for B = 1, 3, 7 and M = 1, 255, 256, 257, 513"""
    L = _L()
    c = L.ctx(cuda)
    slots = sorted({0, 1, PIB_CHUNK - 1, PIB_CHUNK, PIB_CHUNK + 1, 2 * PIB_CHUNK - 1, 2 * PIB_CHUNK, T - 1} & set(range(T)))
    chunks_hit, multi_chunk = set(), 0
    for B in (1, 3, 7):
        for M in (1, 255, 256, 257, 513):
            pts = torch.stack([_pib_points(M, len(slots), 31 * B + M + b)[0] for b in range(B)])
            boxes = torch.stack([_pib_boxes(T, slots, b % 2) for b in range(B)]) if T else torch.zeros((B, 0, 7))
            pib_abi(c, torch.randn((B + 1, M + 300, 3)), torch.rand((B + 1, T + 40, 7)) * 3, 0)   # a larger call first
            got = pib_abi(c, pts, boxes, 0)
            assert torch.equal(got, RA.points_in_boxes_gpu(pts, boxes))
            for b in range(B):
                j = _pib_points(M, len(slots), 31 * B + M + b)[1]
                want = torch.tensor(slots + [-1])[j]
                assert torch.equal(got[b].long(), want)
                if not T:
                    continue
                ins = RA.membership(pts[b], boxes[b])[0]
                in64, near = inbox64(pts[b], boxes[b])
                assert not near.any() and torch.equal(ins, in64)
                first = torch.where(in64.any(0), in64.int().argmax(0), -1)
                assert torch.equal(got[b].long(), first.long())
                chunks_hit |= {int(h) // PIB_CHUNK for h in got[b] if h >= 0}
                lo = torch.where(ins, torch.arange(T)[:, None], T).min(0).values // PIB_CHUNK
                hi = torch.where(ins, torch.arange(T)[:, None], -1).max(0).values // PIB_CHUNK
                multi_chunk += int(((hi > lo) & ins.any(0)).sum())
    assert chunks_hit == set(range((T + PIB_CHUNK - 1) // PIB_CHUNK)), (chunks_hit, T)
    if T > PIB_CHUNK:
        assert multi_chunk > 0, "no point lay in boxes of two chunks"


def test_pib_first_early_exit(cuda):
    """a block whose 255 threads hit in chunk 0 and whose one remaining thread hits only in the last chunk"""
    L = _L()
    c = L.ctx(cuda)
    T = 2 * PIB_CHUNK + 1
    boxes = _pib_boxes(T, [0, T - 1], 0)
    g = torch.Generator().manual_seed(5)
    M = PIB_THREADS + 40
    pts = torch.cat([torch.rand((M, 1), generator=g) * 0.6 - 0.3, torch.rand((M, 2), generator=g) - 0.5], 1)   # in box 0
    lone = 200
    pts[lone, 0] = 1.0                                                                                        # in box T - 1 only
    got = pib_abi(c, pts[None], boxes[None], 0)[0]
    assert torch.equal(got, RA.points_in_boxes_gpu(pts[None], boxes[None])[0])
    assert int(got[lone]) == T - 1 and int(got[lone]) // PIB_CHUNK == (T - 1) // PIB_CHUNK == 2
    others = torch.ones(M, dtype=torch.bool)
    others[lone] = False
    assert (got[others] == 0).all()


def _all_tiles(B, M, T, offset):
    """(alignment of the tile's first element, head, int4 count, tail) of every all-mode tile for `out` at `offset` elements"""
    rows = pib_rows(T)
    res = []
    for b in range(B):
        for row0 in range(0, M, rows):
            base = (b * M + row0) * T
            E = min(rows, M - row0) * T
            a = (offset + base) & 3
            head = min((4 - a) & 3, E)
            nvec = (E - head) >> 2
            res.append((a, head, nvec, E - head - 4 * nvec))
    return res


def test_pib_all_head_alignment_emulation():
    """CPU emulation of the address arithmetic: with the head taken from the element index ((4 - (base & 3)) & 3), an `out` 4, 8 or
    12 bytes past a 16-byte boundary puts every tile's int4 body off its alignment; taken from the address, never"""
    assert "(reinterpret_cast<uintptr_t>(out + base) >> 2) & 3" in RA_SRC
    for T in (1, 3, 5, 31, 33, 257):
        for off_bytes in (0, 4, 8, 12):
            addr = 0x7F0000000000 + off_bytes
            bad_old = bad_new = 0
            for b in range(2):
                for row0 in range(0, 70, pib_rows(T)):
                    base = (b * 70 + row0) * T
                    E = min(pib_rows(T), 70 - row0) * T
                    old = min((4 - (base & 3)) & 3, E)
                    new = min((4 - (((addr + 4 * base) >> 2) & 3)) & 3, E)
                    if (E - old) >> 2:
                        bad_old += (addr + 4 * (base + old)) % 16 != 0
                    if (E - new) >> 2:
                        bad_new += (addr + 4 * (base + new)) % 16 != 0
            assert bad_new == 0
            assert (bad_old > 0) == (off_bytes != 0), (T, off_bytes, bad_old)


def _random_boxes(T, seed, spread=6.0):
    g = torch.Generator().manual_seed(seed)
    xy = (torch.rand((T, 2), generator=g) - 0.5) * 2 * spread
    dims = 0.5 + torch.rand((T, 3), generator=g) * 4
    return torch.cat([xy, -1.5 + torch.rand((T, 1), generator=g), dims, (torch.rand((T, 1), generator=g) - 0.5) * 2 * math.pi], 1)


@pytest.mark.parametrize("T", [1, 3, 5, 31, 32, 33, 257, 12288, 12289, 20000])
def test_pib_all_tiles_and_alignment(cuda, T):
    """every tile's head, int4 body and tail, rows per block from 64 down, and `out` at 0, 4, 8 and 12 bytes"""
    L = _L()
    c = L.ctx(cuda)
    B, M = 2, 70
    rows = pib_rows(T)
    assert M % rows != 0 and rows == (PIB_MAX_ROWS if T <= 12288 else {12289: 63, 20000: 39}[T])
    g = torch.Generator().manual_seed(T)
    pts = torch.cat([(torch.rand((B, M, 2), generator=g) - 0.5) * 12, torch.rand((B, M, 1), generator=g) * 3 - 1.5], 2)
    boxes = torch.stack([_random_boxes(T, T * 3 + b) for b in range(B)])
    boxes[:, 0] = torch.tensor([0.0, 0.0, -2.0, 6.0, 6.0, 4.0, 0.3])
    pib_abi(c, torch.randn((B + 1, M + 64, 3)), torch.rand((B + 1, T, 7)) * 4, 1)   # a larger call first
    exp = torch.stack([RA.membership(pts[b], boxes[b])[0].t() for b in range(B)]).int()
    for b in range(B):
        check_inside(exp[b].t().bool(), pts[b], boxes[b])
    assert exp.any() and not exp.all()
    seen = set()
    for offset in (0, 1, 2, 3):
        got = pib_abi(c, pts, boxes, 1, offset)
        assert torch.equal(got, exp), offset
        tiles = _all_tiles(B, M, T, offset)
        seen |= {t[0] for t in tiles}
        assert any(t[2] > 0 for t in tiles)
        if T % 2:
            assert any(t[1] > 0 for t in tiles) and any(t[3] > 0 for t in tiles)
    if T % 2:
        assert seen == {0, 1, 2, 3}


def test_pib_all_tile_limit(cuda):
    """786432 boxes per sample: one row per block; 786433: refused before any launch"""
    L = _L()
    c = L.ctx(cuda)
    T = PIB_BITS_SMEM // 4 * 32
    assert pib_rows(T) == 1 and pib_rows(T + 1) == 0
    boxes = torch.zeros((1, T, 7))
    boxes[0, :, 0] = 1000.0 + torch.arange(T).float() * 1e-2
    boxes[0, :, 3:6] = 1.0
    for k in (0, 1, T // 2, T - 1):
        boxes[0, k] = torch.tensor([float(k % 3), 0.0, -1.0, 0.8, 0.8, 2.0, 0.2 * k])
    pts = torch.tensor([[[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [2.0, -0.1, 0.5]]])
    got = pib_abi(c, pts, boxes, 1)
    exp = RO.box_test(pts[0], boxes[0])[0]
    assert torch.equal(got[0].t().bool(), exp) and int(exp.sum()) == 4
    buf = torch.full((8,), ISENT, dtype=torch.int32, device="cuda")
    b2 = torch.zeros((1, T + 1, 7), device="cuda")
    p2 = pts.cuda()
    assert L.lib().sstb200_points_in_boxes(c, p2.data_ptr(), b2.data_ptr(), 1, 1, T + 1, 1, buf.data_ptr()) == ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert (buf.cpu() == ISENT).all()


# ---- dynamic_point_pool through the C ABI ------------------------------------------------------------------------------------------
def dpp_abi(c, rois, pts, max_inbox, max_all, rb=None, pb=None, per_sample=0, nsamp=1, extra=EXTRA, expect=0):
    """outputs of max_all (x nsamp per sample) rows pre-filled with sentinels, GUARD rows past them; returns idx, roi, feats, host[3]"""
    L = _L()
    cap = max_all * (nsamp if per_sample else 1)
    idx = torch.full((cap + GUARD,), ISENT, dtype=torch.int64, device="cuda")
    roi = torch.full((cap + GUARD,), ISENT, dtype=torch.int64, device="cuda")
    feats = torch.full(((cap + GUARD) * 13,), FSENT, dtype=torch.int32, device="cuda")
    num = torch.full((1,), ISENT, dtype=torch.int32, device="cuda")
    host = (C.c_int32 * 3)()
    r, p = rois.float().contiguous().cuda(), pts.float().contiguous().cuda()
    rbc = None if rb is None else rb.int().contiguous().cuda()
    pbc = None if pb is None else pb.int().contiguous().cuda()
    rc = L.lib().sstb200_dynamic_point_pool(c, r.data_ptr(), L.ptr(rbc), r.shape[0], p.data_ptr(), L.ptr(pbc), p.shape[0],
                                            L.arr(C.c_float, [float(v) for v in extra]), int(max_inbox), int(max_all), int(per_sample),
                                            idx.data_ptr(), roi.data_ptr(), feats.data_ptr(), num.data_ptr(), host)
    if expect:
        assert rc == expect, (rc, L.lib().sstb200_last_error(c))
        return None
    assert rc == 0, L.lib().sstb200_last_error(c)
    k = host[0]
    assert int(num.item()) == k and 0 < k <= cap
    idx, roi, feats = idx.cpu(), roi.cpu(), feats.cpu()
    assert (idx[k:] == ISENT).all() and (roi[k:] == ISENT).all() and (feats[k * 13:] == FSENT).all(), "a row past the count was written"
    assert (idx[:k] != ISENT).all() and (roi[:k] != ISENT).all() and (feats[:k * 13] != FSENT).all(), "a row was not fully written"
    return idx[:k], roi[:k], feats[:k * 13].view(torch.float32).view(k, 13), tuple(host)


def dpp_poison(c):
    pts, rois, _, _ = RO.synth_roi_frame(99, n_pts=30000, n_rois=300, spread=20.0)
    dpp_abi(c, rois, pts * 1e3, 512, 60000)


def dpp_expect(rois, pts, max_inbox, max_all, rb=None, pb=None, cand=None, extra=EXTRA):
    """the oracle over the candidate points only (the others lie far outside every enlarged RoI), indices mapped back"""
    sub = pts if cand is None else pts[cand]
    psub = None if pb is None else (pb if cand is None else pb[cand])
    i, r, f = RO.dynamic_point_pool(rois, sub, extra, max_inbox, max_all_pts=10 ** 9, rois_batch=rb, pts_batch=psub)
    if cand is not None and i[0] >= 0:
        i = cand[i]
    return i[:max_all], r[:max_all], f[:max_all]


def check_feats64(got, rois, pts_of):
    """raw xyz bitwise, local xyz and the six boundary offsets against float64 within the kernel's fp32 error"""
    idx, roi, feats = got[0], got[1], got[2]
    real = idx >= 0
    if not real.any():
        return
    p = pts_of(idx[real]).float()
    assert torch.equal(_bits(feats[real, :3]), _bits(p))
    b = rois[roi[real]].double()
    lx, ly, dz, exy, ez = _local64(p.double(), b)
    hl, hw, hh = b[:, 4] / 2, b[:, 3] / 2, b[:, 5] / 2
    ref = torch.stack([lx, ly, dz, hl + lx, hw + ly, hh + dz, hl - lx, hw - ly, hh - dz], 1)
    eo = lambda e, h, v: e + 2 * U * (h.abs() + v.abs())
    bound = torch.stack([exy, exy, ez, eo(exy, hl, lx), eo(exy, hw, ly), eo(ez, hh, dz), eo(exy, hl, lx), eo(exy, hw, ly), eo(ez, hh, dz)], 1)
    g = feats[real, 3:12].double()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isnan(g), torch.isnan(ref))
    err = (g - ref).abs()
    bad = fin & (err > bound)
    assert not bad.any(), f"local features off float64 by {err[bad][:4].tolist()} > {bound[bad][:4].tolist()}"


def check_dpp(got, exp, rois, pts_of, members=None):
    """idx, roi and is_in_margin exact against the fp32 oracle, features against float64; members = (pts, cand): also the pair set
    against the float64 in-box test of the enlarged RoIs (only when nothing was cut)"""
    assert torch.equal(got[0], exp[0]) and torch.equal(got[1], exp[1]), (got[0][:8], exp[0][:8])
    assert torch.equal(_bits(got[2][:, :3]), _bits(exp[2][:, :3])) and torch.equal(got[2][:, 12], exp[2][:, 12])
    check_feats64(got, rois, pts_of)
    if members is not None:
        sub, cand = members
        big = RO.enlarge_boxes(rois, EXTRA)
        inside = torch.zeros((rois.shape[0], sub.shape[0]), dtype=torch.bool)
        real = got[0] >= 0
        pos = torch.searchsorted(cand, got[0][real])
        inside[got[1][real], pos] = True
        return check_inside(inside, sub, big)


FILL_X, FILL_Y = 2000.0, -3000.0


def filler(n, seed):
    """n points on the GPU in [2000, 3000] x [-3000, -2000]: outside every RoI of these tests"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand((n, 3), device="cuda", generator=g) * 1000 + torch.tensor([FILL_X, FILL_Y, -500.0], device="cuda")


def _far_from_filler(rois):
    r = (rois[:, 3].abs() + rois[:, 4].abs() + 2).max()
    assert ((rois[:, 0] + r < FILL_X) | (rois[:, 1] - r > FILL_Y + 1000)).all()


# ---- dynamic_point_pool: radix-select passes and take sizes ---------------------------------------------------------------------
@pytest.mark.parametrize("n_pts", [256, 257, 65536, 65537, 1 << 24, (1 << 24) + 1])
def test_dpp_radix_passes(cuda, n_pts):
    """RoI 0 holds indices that share their low bytes and differ only in the top radix digit; RoI 1 random indices"""
    L = _L()
    c = L.ctx(cuda)
    passes = radix_passes(n_pts)
    assert passes == {256: 1, 257: 2, 65536: 2, 65537: 3, 1 << 24: 3, (1 << 24) + 1: 4}[n_pts]
    top = 8 * (passes - 1)
    a_idx = torch.arange(0, n_pts, 1 << top) if top else torch.arange(0, n_pts, 2)
    assert a_idx.numel() >= 2 and (a_idx % (1 << top) == 0).all() and ((a_idx[1:] >> top) != (a_idx[:-1] >> top)).all()
    g = torch.Generator().manual_seed(n_pts % 1000)
    rest = torch.tensor(sorted(set(range(n_pts)) - set(a_idx.tolist()))) if n_pts < 70000 else torch.randint(0, n_pts, (4000,), generator=g)
    b_idx = torch.unique(rest[torch.randperm(rest.numel(), generator=g)[:600]])
    b_idx = b_idx[~torch.isin(b_idx, a_idx)]
    cand = torch.cat([a_idx, b_idx]).sort()[0]
    rois = torch.tensor([[0.0, 0.0, -1.0, 2.0, 2.0, 2.0, 0.4], [10.0, 0.0, -1.0, 3.0, 3.0, 2.0, -0.7]])
    _far_from_filler(rois)
    sub = torch.zeros((cand.numel(), 3))
    ina = torch.isin(cand, a_idx)
    sub[ina] = (torch.rand((int(ina.sum()), 3), generator=g) - 0.5) * torch.tensor([1.2, 1.2, 1.5])
    sub[~ina] = (torch.rand((int((~ina).sum()), 3), generator=g) - 0.5) * torch.tensor([2.0, 2.0, 1.5]) + torch.tensor([10.0, 0.0, 0.0])
    pts = filler(n_pts, n_pts % 997)
    pts[cand.cuda()] = sub.cuda()
    pts_of = lambda i: sub[torch.searchsorted(cand, i)]
    hits_a = a_idx.numel()
    for take in sorted({1, 2, 255, 256, 257, max(hits_a - 1, 1)}):
        dpp_poison(c)
        got = dpp_abi(c, rois, pts, take, 10 ** 5)
        check_dpp(got, _dpp_expect_sub(rois, sub, cand, take), rois, pts_of)
        kept_a = got[0][got[1] == 0]
        assert kept_a.numel() == min(take, hits_a) and torch.equal(kept_a, a_idx[:take])
        assert (got[1] == 1).sum() == min(take, b_idx.numel())
    assert hits_a > 1 and b_idx.numel() > 100


def _dpp_expect_sub(rois, sub, cand, take):
    i, r, f = RO.dynamic_point_pool(rois, sub, EXTRA, take, max_all_pts=10 ** 9)
    return (cand[i] if i[0] >= 0 else i), r, f


def test_dpp_take_sizes(cuda):
    """take = 1 .. 8192 around every power of two the bitonic sort pads to; 8193 refused"""
    L = _L()
    c = L.ctx(cuda)
    g = torch.Generator().manual_seed(8)
    n_big = 9000
    big = (torch.rand((n_big, 3), generator=g) - 0.5) * torch.tensor([28.0, 18.0, 2.0])
    mid = (torch.rand((300, 3), generator=g) - 0.5) * torch.tensor([1.5, 1.5, 1.0]) + torch.tensor([40.0, 0.0, 0.0])
    bg = (torch.rand((3000, 3), generator=g) - 0.5) * 200
    pts = torch.cat([big, mid, bg])[torch.randperm(n_big + 3300, generator=g)]
    rois = torch.tensor([[0.0, 0.0, -1.5, 20.0, 30.0, 3.0, math.pi / 2], [40.0, 0.0, -1.0, 2.0, 2.0, 2.0, 0.3],
                         [-60.0, 60.0, -1.0, 4.0, 4.0, 3.0, 1.0]])
    assert table_size(pts.shape[0]) > footprint_cells(rois[0].tolist(), EXTRA)       # the hashed route
    dense = RO.dynamic_point_pool(rois, pts, EXTRA, RP_MAX_INBOX, max_all_pts=10 ** 9)
    assert (dense[1] == 0).sum() == RP_MAX_INBOX
    for take in (1, 2, 255, 256, 257, 4095, 4096, 4097, 8191, 8192):
        dpp_poison(c)
        got = dpp_abi(c, rois, pts, take, 10 ** 5)
        check_dpp(got, dpp_expect(rois, pts, take, 10 ** 5), rois, lambda i: pts[i])
        assert (got[1] == 0).sum() == take and got[3][1] > take
    dpp_abi(c, rois, pts, RP_MAX_INBOX + 1, 10 ** 5, expect=ERR_UNSUPPORTED)
    dpp_abi(c, rois, pts, 0, 10 ** 5, expect=ERR_ARG)


def _sample_frame(seed, nsamp, empty):
    """nsamp samples, sample-sorted RoIs; the samples in `empty` have RoIs but no pair"""
    pts, rois, pb, rb = RO.synth_roi_frame(seed, n_pts=6000, n_rois=60, spread=12.0, batch_size=nsamp)
    for s in empty:
        rois[rb == s, 0] += 400.0
    return pts, rois, pb, rb


def _per_sample_expect(pts, rois, pb, rb, take, max_all):
    parts = []
    for s in sorted(set(rb.tolist())):
        rm, pm = rb == s, pb == s
        pidx, ridx = pm.nonzero()[:, 0], rm.nonzero()[:, 0]
        i, r, f = RO.dynamic_point_pool(rois[rm], pts[pm], EXTRA, take, max_all_pts=max_all)
        if i[0] >= 0:
            i, r = pidx[i], ridx[r]
        else:
            assert r[0] == -1
        parts.append((i, r, f))
    return tuple(torch.cat([p[k] for p in parts]) for k in range(3))


@pytest.mark.parametrize("empty", [(0,), (2,), (4,), (0, 2, 4)])
def test_dpp_capacity_and_fake_rows(cuda, empty):
    """max_all_pts mid-RoI, on a RoI boundary, on the last pair and one before it, per call and per sample; fake rows for the empty
    samples wherever they sit"""
    L = _L()
    c = L.ctx(cuda)
    pts, rois, pb, rb = _sample_frame(21 + len(empty) + empty[0], 5, empty)
    take = 32
    full = dpp_expect(rois, pts, take, 10 ** 9, rb=rb, pb=pb)
    per_roi = torch.bincount(full[1][full[1] >= 0], minlength=rois.shape[0])
    cum = per_roi.cumsum(0)
    r_mid = int((per_roi > 3).nonzero()[1])
    total = int(cum[-1])
    for max_all in (int(cum[r_mid]) - 2, int(cum[r_mid]), total - 1, total):
        dpp_poison(c)
        got = dpp_abi(c, rois, pts, take, max_all, rb=rb, pb=pb)
        exp = dpp_expect(rois, pts, take, max_all, rb=rb, pb=pb)
        check_dpp(got, exp, rois, lambda i: pts[i])
        assert got[3][1] == total and got[3][2] == min(max_all, total)
    sample_pairs = [int(per_roi[rb == s].sum()) for s in range(5)]
    assert all(sample_pairs[s] == 0 for s in empty) and all(sample_pairs[s] > 0 for s in range(5) if s not in empty)
    nonempty = [s for s in range(5) if s not in empty]
    pr = per_roi[rb == nonempty[0]]
    first = int(pr[pr > 0][0])                                                 # the first RoI boundary of that sample
    least = min(sample_pairs[s] for s in nonempty)
    for max_all in (3, first, least - 1, least, max(sample_pairs)):
        dpp_poison(c)
        got = dpp_abi(c, rois, pts, take, max_all, rb=rb, pb=pb, per_sample=1, nsamp=5)
        exp = _per_sample_expect(pts, rois, pb, rb, take, max_all)
        check_dpp(got, exp, rois, lambda i: pts[i])
        fake = (got[0] == -1).nonzero()[:, 0].tolist()
        assert len(fake) == len(empty) and (got[2][fake] == 0).all()
        assert got[3][0] - got[3][2] == len(empty)


def test_dpp_refusals(cuda):
    """per-sample RoIs out of batch order and negative batch ids are refused"""
    L = _L()
    c = L.ctx(cuda)
    pts, rois, pb, rb = _sample_frame(31, 3, ())
    dpp_abi(c, rois.flip(0), pts, 16, 1000, rb=rb.flip(0), pb=pb, per_sample=1, nsamp=3, expect=ERR_ARG)
    bad = rb.clone()
    bad[5] = -1
    dpp_abi(c, rois, pts, 16, 1000, rb=bad, pb=pb, expect=ERR_ARG)
    badp = pb.clone()
    badp[7] = -2
    dpp_abi(c, rois, pts, 16, 1000, rb=rb, pb=badp, expect=ERR_ARG)
    got = dpp_abi(c, rois.flip(0), pts, 16, 10 ** 5, rb=rb.flip(0), pb=pb)     # unsorted is fine when capacity is per call
    check_dpp(got, dpp_expect(rois.flip(0), pts, 16, 10 ** 5, rb=rb.flip(0), pb=pb), rois.flip(0), lambda i: pts[i])


@pytest.mark.parametrize("take", [1, 255, 256, 257])
def test_dpp_mixed_vs_per_sample_calls(cuda, take):
    L = _L()
    c = L.ctx(cuda)
    pts, rois, pb, rb = _sample_frame(41 + take, 3, (1,))
    rois[3, 3:5] = 24.0
    assert int(rb[3]) == 0 and int(RA.membership(pts[pb == 0], RO.enlarge_boxes(rois[3:4], EXTRA))[0].sum()) > take   # hits > take
    got = dpp_abi(c, rois, pts, take, 10 ** 6, rb=rb, pb=pb)
    parts = []
    for s in range(3):
        rm, pm = rb == s, pb == s
        i, r, f, _ = dpp_abi(c, rois[rm], pts[pm], take, 10 ** 6)
        if i[0] >= 0:
            parts.append((pm.nonzero()[:, 0][i], rm.nonzero()[:, 0][r], f))
    for k in range(3):
        assert torch.equal(got[k], torch.cat([p[k] for p in parts]))
    assert ((got[1] == 3).sum() == take) and torch.equal(rb[got[1]], pb[got[0]])


# ---- the BEV grid, through dynamic_point_pool and RoIAwarePool3d --------------------------------------------------------------------
def ra_plan(c, rois, pts, out_size, m, rb=None, pb=None):
    L = _L()
    P = C.c_int64(-7)
    r = rois.float().contiguous().cuda()
    p = pts.float().contiguous().cuda()
    rbc = None if rb is None else rb.int().contiguous().cuda()
    pbc = None if pb is None else pb.int().contiguous().cuda()
    rc = L.lib().sstb200_roiaware_pool3d_plan(c, r.data_ptr(), L.ptr(rbc), r.shape[0], p.data_ptr(), L.ptr(pbc), p.shape[0],
                                              L.arr(C.c_int32, list(out_size)), int(m), C.byref(P))
    return rc, P.value


def ra_forward(c, rois, pts, feats, out_size, m, mode, rb=None, pb=None):
    """plan + forward into sentinel-filled outputs with guard space; returns pooled [R, ox, oy, oz, C] and the state"""
    L = _L()
    rois, pts = rois.float().contiguous().cuda(), pts.float().contiguous().cuda()      # the plan keeps these pointers for the forward
    rb = None if rb is None else rb.int().contiguous().cuda()
    pb = None if pb is None else pb.int().contiguous().cuda()
    rc, P = ra_plan(c, rois, pts, out_size, m, rb, pb)
    assert rc == 0 and P >= 0, L.lib().sstb200_last_error(c)
    R, Ch = rois.shape[0], feats.shape[1]
    nvox = out_size[0] * out_size[1] * out_size[2]
    n = R * nvox * Ch
    P1 = max(P, 1)
    pooled = torch.full((n + GUARD,), FSENT, dtype=torch.int32, device="cuda")
    slot = torch.full((P1 + GUARD,), ISENT, dtype=torch.int64, device="cuda")
    voff = torch.full((P + 1 + GUARD,), ISENT, dtype=torch.int32, device="cuda")
    pidx = torch.full((P1 + GUARD,), ISENT, dtype=torch.int32, device="cuda")
    argmax = torch.full(((P1 + GUARD) * Ch,), ISENT, dtype=torch.int32, device="cuda") if mode == 0 else None
    counts = torch.full((2 + GUARD,), ISENT, dtype=torch.int32, device="cuda")
    f = feats.float().contiguous().cuda()
    rc = L.lib().sstb200_roiaware_pool3d_forward(c, f.data_ptr(), Ch, mode, pooled.data_ptr(), slot.data_ptr(), voff.data_ptr(),
                                                 pidx.data_ptr(), L.ptr(argmax), counts.data_ptr())
    assert rc == 0, L.lib().sstb200_last_error(c)
    cnt = counts.cpu()
    V, K = int(cnt[0]), int(cnt[1])
    assert (cnt[2:] == ISENT).all() and 0 <= V <= P and 0 <= K <= P
    pc, sc, vc, ic = pooled.cpu(), slot.cpu(), voff.cpu(), pidx.cpu()
    assert (pc[n:] == FSENT).all() and (pc[:n] != FSENT).all()
    assert (sc[P1:] == ISENT).all() and (sc[:V] != ISENT).all()
    assert (vc[P + 1:] == ISENT).all() and (vc[:V + 1] != ISENT).all() and int(vc[V]) == K
    assert (ic[P1:] == ISENT).all() and (ic[:K] != ISENT).all()
    if mode == 0:
        ac = argmax.cpu()
        assert (ac[P1 * Ch:] == ISENT).all() and (ac[:V * Ch] != ISENT).all()
    state = (slot, voff, pidx, argmax, counts, P)
    return pc[:n].view(torch.float32).view(R, *out_size, Ch), state


def ra_backward(c, state, N, Ch, mode, grad):
    L = _L()
    slot, voff, pidx, argmax, counts, P = state
    gin = torch.full(((N + 4) * Ch,), FSENT, dtype=torch.int32, device="cuda")
    g = grad.float().contiguous().cuda()
    rc = L.lib().sstb200_roiaware_pool3d_backward(c, N, Ch, mode, P, slot.data_ptr(), voff.data_ptr(), pidx.data_ptr(), L.ptr(argmax),
                                                  counts.data_ptr(), g.data_ptr(), gin.data_ptr())
    assert rc == 0, L.lib().sstb200_last_error(c)
    gin = gin.cpu()
    assert (gin[N * Ch:] == FSENT).all() and (gin[:N * Ch] != FSENT).all()
    return gin[:N * Ch].view(torch.float32).view(N, Ch)


def ra_poison(c):
    pts, rois, _, _ = RO.synth_roi_frame(98, n_pts=20000, n_rois=80, spread=10.0)
    feats = torch.randn((pts.shape[0], 40)) * 1e3
    pooled, st = ra_forward(c, rois, pts, feats, (7, 6, 5), 200, 0)
    ra_backward(c, st, pts.shape[0], 40, 0, torch.randn(pooled.shape))


def ra_expect(rois, pts, feats, out_size, m, mode, rb=None, pb=None, cand=None):
    """the oracle over the candidate points, point indices mapped back"""
    sub, fs = (pts, feats) if cand is None else (pts[cand], feats[cand])
    psub = None if pb is None else (pb if cand is None else pb[cand])
    pooled, arg, pidx = RA.roiaware_pool3d(rois, sub, fs, out_size, m, mode, rois_batch=rb, pts_batch=psub)
    if cand is not None:
        body = pidx[..., 1:]
        used = torch.arange(m - 1) < pidx[..., :1]
        body[used] = cand[body[used].long()].int()
        arg = torch.where(arg >= 0, cand[arg.clamp(min=0).long()].int(), arg)
    return pooled, arg, pidx


def bwd_emulate(dense_idx, dense_arg, grad, N, mode):
    """the backward's sum for every (point, channel): its terms in (roi, voxel) order added one by one in fp32; also the float64
    sum, sum |term| and the number of terms per point"""
    Ch, m = grad.shape[-1], dense_idx.shape[-1]
    pi = dense_idx.reshape(-1, m).long()
    cnt = pi[:, 0]
    g = grad.reshape(-1, Ch).float()
    v, s = (torch.arange(m - 1)[None] < cnt[:, None]).nonzero(as_tuple=True)   # slot-major: (roi, voxel) order
    pt = pi[v, s + 1]
    if mode == 0:
        sel = dense_arg.reshape(-1, Ch)[v].long() == pt[:, None]
        t32 = torch.where(sel, g[v], torch.zeros_like(g[v]))
        t64 = t32.double()
    else:
        cur = torch.ones(cnt.shape) / cnt.clamp(min=1).float()
        t32 = g[v] * cur[v][:, None]
        t64 = g[v].double() / cnt[v].clamp(min=1).double()[:, None]
    order = torch.sort(pt, stable=True).indices
    pt, t32, t64 = pt[order], t32[order], t64[order]
    k = torch.bincount(pt, minlength=N)
    start = torch.repeat_interleave(k.cumsum(0) - k, k)
    rank = torch.arange(pt.numel()) - start
    acc = torch.zeros((N, Ch))
    for j in range(int(k.max()) if pt.numel() else 0):
        sel = rank == j
        acc[pt[sel]] = acc[pt[sel]] + t32[sel]
    s64 = torch.zeros((N, Ch), dtype=torch.float64).index_add_(0, pt, t64)
    a64 = torch.zeros((N, Ch), dtype=torch.float64).index_add_(0, pt, t64.abs())
    return acc, s64, a64, k


def check_pool(c, rois, pts, feats, out_size, m, mode, rb=None, pb=None, cand=None, grad=True, poison=True):
    """forward bitwise against the oracle (state expanded to the reference's dense layout), avg within float64 bounds, kept points
    against float64 membership; backward bitwise against the emulation, within float64 bounds, run to run"""
    if poison:
        ra_poison(c)
    R, N, Ch = rois.shape[0], pts.shape[0], feats.shape[1]
    pooled, st = ra_forward(c, rois, pts, feats, out_size, m, mode, rb, pb)
    e_pooled, e_arg, e_pidx = ra_expect(rois, pts, feats, out_size, m, mode, rb, pb, cand)
    slot, voff, pidx, argmax, counts, P = st
    dense_idx, dense_arg = RA.expand_state(slot.cpu(), voff.cpu(), pidx.cpu(), None if argmax is None else argmax.cpu().view(-1, Ch),
                                           counts.cpu(), R, out_size, m, Ch)
    assert torch.equal(_bits(pooled), _bits(e_pooled))
    assert torch.equal(dense_idx, e_pidx)
    if mode == 0:
        assert torch.equal(dense_arg, e_arg)
    else:
        cnt = dense_idx.reshape(-1, m)[:, 0].long()
        occ = (cnt > 0).nonzero()[:, 0]
        if occ.numel():
            pi = dense_idx.reshape(-1, m)[occ, 1:].long()
            use = (torch.arange(m - 1)[None] < cnt[occ][:, None])[..., None]
            fx = torch.where(use, feats.cpu()[pi].double(), torch.zeros((), dtype=torch.float64))
            mean = fx.sum(1) / cnt[occ].double()[:, None]
            bound = cnt[occ].double()[:, None] * U * fx.abs().sum(1)
            got = pooled.reshape(-1, Ch)[occ].double()
            fin = torch.isfinite(mean)
            assert ((got - mean).abs()[fin] <= bound[fin]).all()
    if grad:
        g = torch.randn(pooled.shape, generator=torch.Generator().manual_seed(R + N)) * \
            10.0 ** torch.randint(-3, 4, pooled.shape, generator=torch.Generator().manual_seed(3)).float()
        gin = ra_backward(c, st, N, Ch, mode, g)
        assert torch.equal(_bits(gin), _bits(ra_backward(c, st, N, Ch, mode, g)))
        acc, s64, a64, k = bwd_emulate(dense_idx, dense_arg, g, N, mode)
        assert torch.equal(_bits(gin), _bits(acc))
        bound = (k.double()[:, None] + 2) * U * a64
        assert ((gin.double() - s64).abs() <= bound).all()
    return pooled, st, dense_idx


def _box_corners(roi, eps_steps=(-4, -1, 0, 1, 4)):
    """points a few fp32 steps either side of each BEV corner of the box (world coordinates), at mid height"""
    cx, cy, zb, w, l, h, rz = roi
    ang = rz + math.pi / 2
    ca, sa = math.cos(ang), math.sin(ang)
    out = []
    for ux, uy in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
        lx, ly = ux * l / 2, uy * w / 2
        x, y = np.float32(cx + lx * ca + ly * sa), np.float32(cy - lx * sa + ly * ca)
        for dx in eps_steps:
            for dy in eps_steps:
                xs = x
                ys = y
                for _ in range(abs(dx)):
                    xs = np.nextafter(xs, np.float32(np.inf if dx > 0 else -np.inf))
                for _ in range(abs(dy)):
                    ys = np.nextafter(ys, np.float32(np.inf if dy > 0 else -np.inf))
                out.append([float(xs), float(ys), zb + h / 2])
    return out


def _far_case(X, Y, seed):
    """RoIs around (X, Y) at yaw 0, 45 deg and one fp32 step off it, a 40 m RoI, a negative-dims RoI; points in them, a few fp32
    steps either side of every corner, on integer cell boundaries, with NaN x / y and a NaN z"""
    g = torch.Generator().manual_seed(seed)
    q = math.pi / 4
    q1 = float(np.nextafter(np.float32(q), np.float32(1)))
    rois = [[X, Y, -1.0, 2.0, 4.0, 2.0, 0.0], [X + 7.0, Y, -1.0, 1.6, 3.2, 2.0, q], [X, Y + 7.0, -1.0, 1.6, 3.2, 2.0, q1],
            [X - 7.0, Y - 3.0, -1.0, 1.0, 1.0, 2.0, -q], [X + 20.0, Y + 20.0, -1.0, 40.0, 40.0, 3.0, 0.3],
            [X - 9.0, Y + 9.0, -1.0, -2.0, 3.0, 2.0, 0.0], [X - 12.0, Y - 12.0, -1.0, 3.0, 3.0, -1.0, 0.0]]
    rois = [[float(np.float32(v)) for v in r] for r in rois]
    pts = []
    for r in rois:
        if r[3] > 0 and r[5] > 0:
            pts += _box_corners(r)
            if r[3] < 10:
                big = RO.enlarge_boxes(torch.tensor([r]), EXTRA)[0].tolist()
                pts += _box_corners(big)
    for r in rois[:4]:
        base = np.floor(np.float32(r[0])), np.floor(np.float32(r[1]))
        for i in range(-3, 4):
            for j in range(-3, 4):
                pts.append([float(base[0] + i), float(base[1] + j), 0.0])
    inner = (torch.rand((400, 3), generator=g) - 0.5) * torch.tensor([44.0, 44.0, 2.0]) + torch.tensor([X + 20.0, Y + 20.0, 0.5])
    near = (torch.rand((400, 3), generator=g) - 0.5) * torch.tensor([30.0, 30.0, 2.5]) + torch.tensor([X, Y, 0.0])
    nan = torch.tensor([[float("nan"), Y, 0.0], [X, float("nan"), 0.0], [float("nan"), float("nan"), 0.0], [X, Y, float("nan")],
                        [X - 9.0, Y + 9.0, 0.0], [X - 12.0, Y - 12.0, -1.0]])
    pts = torch.cat([torch.tensor(pts, dtype=torch.float32), inner.float(), near.float(), nan])
    pts = pts[torch.randperm(pts.shape[0], generator=g)]
    return torch.tensor(rois, dtype=torch.float32), pts


@pytest.mark.parametrize("X,Y", [(0.0, 0.0), (1e4, -1e4), (-3.3e4, 3.3e4), (1e5, 1e5), (-1e5, -3.3e4)])
def test_grid_far_coordinates(cuda, X, Y):
    """corners, cell boundaries, 45 deg, NaN and negative dims, near the origin, at 1e4 m, past the cell clamp and at 1e5 m"""
    L = _L()
    c = L.ctx(cuda)
    rois, pts = _far_case(X, Y, int(abs(X) + abs(Y)) % 1000 + 1)
    N = pts.shape[0]
    cand = torch.arange(N)
    if abs(X) > CELL_CLAMP or abs(Y) > CELL_CLAMP:
        assert cell(X) in (-CELL_CLAMP, CELL_CLAMP) or cell(Y) in (-CELL_CLAMP, CELL_CLAMP)
    dpp_poison(c)
    got = dpp_abi(c, rois, pts, RP_MAX_INBOX, 10 ** 6)
    clear = check_dpp(got, dpp_expect(rois, pts, RP_MAX_INBOX, 10 ** 6), rois, lambda i: pts[i], members=(pts, cand))
    assert clear > 0
    nan_xy = torch.isnan(pts[:, 0]) | torch.isnan(pts[:, 1])
    assert not torch.isin(got[0], nan_xy.nonzero()[:, 0]).any()
    assert not ((got[1] == 5) | (got[1] == 6)).any()                         # negative w, negative h: empty
    admitted_corner = 0
    for r in range(4):
        mine = got[0][got[1] == r]
        big = RO.enlarge_boxes(rois[r:r + 1], EXTRA)[0].tolist()
        cs = torch.tensor(_box_corners(big, (-1, 0, 1)))
        hit = (pts[mine][:, None, :2] == cs[None, :, :2]).all(2).any(0)
        admitted_corner += int(hit.sum())
    assert admitted_corner > 0, "no point one fp32 step from a corner was admitted"
    for mode in (0, 1):
        feats = torch.randn((N, 5), generator=torch.Generator().manual_seed(mode))
        pooled, st, dense = check_pool(c, rois, pts, feats, (4, 3, 2), 64, mode)
        assert int(st[4][0].item()) > 0
    assert torch.isnan(pts[:, 2]).any()


def test_grid_footprint_fallback(cuda):
    """a 40 m x 40 m RoI over 512 points takes the every-point route, over 2000 points the hashed route: the same pairs"""
    L = _L()
    c = L.ctx(cuda)
    roi = torch.tensor([[3.0, -2.0, -2.0, 40.0, 40.0, 4.0, 0.6], [30.0, 30.0, -1.0, 2.0, 2.0, 2.0, 0.0]])
    nc = footprint_cells(roi[0].tolist(), EXTRA)
    assert nc > table_size(512) and nc <= table_size(2000)
    g = torch.Generator().manual_seed(12)
    pts = (torch.rand((512, 3), generator=g) - 0.5) * torch.tensor([70.0, 70.0, 5.0])
    more = torch.cat([pts, filler(2000 - 512, 3).cpu()])
    res = []
    for p in (pts, more):
        dpp_poison(c)
        got = dpp_abi(c, roi, p, RP_MAX_INBOX, 10 ** 5)
        check_dpp(got, dpp_expect(roi, pts, RP_MAX_INBOX, 10 ** 5, cand=torch.arange(512)), roi, lambda i: pts[i],
                  members=(pts, torch.arange(512)))
        res.append(got)
        feats = torch.randn((p.shape[0], 3), generator=torch.Generator().manual_seed(4))
        check_pool(c, roi, p, feats, (5, 5, 3), 16, 1, cand=torch.arange(512) if p is more else None)
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1]) and int((res[0][1] == 0).sum()) > 100


@pytest.mark.parametrize("N", [512, 513, (1 << 23) + 1])
def test_grid_table_sizes(cuda, N):
    """the bucket table doubles at N = 512 | 513 and stops at 2^24 buckets"""
    L = _L()
    c = L.ctx(cuda)
    assert table_size(N) == {512: 1024, 513: 2048, (1 << 23) + 1: 1 << 24}[N]
    g = torch.Generator().manual_seed(N % 1000)
    rois = _random_boxes(40, N % 777, spread=15.0)
    rois[:, 3:6] = rois[:, 3:6].clamp(max=3.0)
    _far_from_filler(rois)
    ncand = min(N, 500)
    cand = torch.sort(torch.randperm(N, generator=g)[:ncand])[0]
    sub = torch.cat([(torch.rand((ncand, 2), generator=g) - 0.5) * 34, torch.rand((ncand, 1), generator=g) * 3 - 1.5], 1)
    pts = filler(N, 7)
    pts[cand.cuda()] = sub.cuda()
    pts_of = lambda i: sub[torch.searchsorted(cand, i)]
    dpp_poison(c)
    got = dpp_abi(c, rois, pts, RP_MAX_INBOX, 10 ** 5)
    exp = _dpp_expect_sub(rois, sub, cand, RP_MAX_INBOX)
    check_dpp(got, exp, rois, pts_of, members=(sub, cand))
    assert got[0].numel() > 20
    feats_sub = torch.randn((ncand, 4), generator=g)
    feats = torch.zeros((N, 4), device="cuda")
    feats[cand.cuda()] = feats_sub.cuda()
    for mode in (0, 1):
        ra_poison(c)
        pooled, st = ra_forward(c, rois, pts, feats, (3, 4, 2), 32, mode)
        e_pooled, e_arg, e_pidx = RA.roiaware_pool3d(rois, sub, feats_sub, (3, 4, 2), 32, mode)
        slot, voff, pidx, argmax, counts, P = st
        dense_idx, dense_arg = RA.expand_state(slot.cpu(), voff.cpu(), pidx.cpu(), None if argmax is None else argmax.cpu().view(-1, 4),
                                               counts.cpu(), rois.shape[0], (3, 4, 2), 32, 4)
        body, used = e_pidx[..., 1:], torch.arange(31) < e_pidx[..., :1]
        body[used] = cand[body[used].long()].int()
        assert torch.equal(_bits(pooled), _bits(e_pooled)) and torch.equal(dense_idx, e_pidx)
        if mode == 0:
            assert torch.equal(dense_arg, torch.where(e_arg >= 0, cand[e_arg.clamp(min=0).long()].int(), e_arg))


def test_grid_hash_collisions(cuda):
    """(cell, batch) triples that share a bucket, across cells of one batch and across batches: no point admitted twice or across
    batches"""
    L = _L()
    c = L.ctx(cuda)
    n_target = 600
    mask = table_size(n_target) - 1
    h0 = bucket(10, 10, 0, mask)
    xs, ys = np.meshgrid(np.arange(-60, 61), np.arange(-60, 61), indexing="ij")
    found = {}
    for b in (0, 1, 2):
        hs = np.array([[bucket(int(x), int(y), b, mask) for y in range(-60, 61)] for x in range(-60, 61)])
        for x, y in zip(xs[hs == h0], ys[hs == h0]):
            if (int(x), int(y), b) != (10, 10, 0):
                found.setdefault(b, []).append((int(x), int(y)))
    assert len(found.get(0, [])) >= 1 and len(found.get(1, [])) >= 1, found
    # batch id mask + 1 puts cell (10, 10) in the same bucket as batch 0 with the same cell key: only the batch test separates them
    big_b = mask + 1
    cells = [(10, 10, 0), (*found[0][0], 0), (*found[1][0], 1), (10, 10, big_b), (10, 10, 1)] + \
        ([(*found[2][0], 2)] if found.get(2) else [])
    assert len({bucket(x, y, b, mask) for x, y, b in cells[:4]}) == 1
    g = torch.Generator().manual_seed(77)
    pts, pb, rois, rb = [], [], [], []
    for x, y, b in cells:
        pts.append(torch.rand((40, 3), generator=g) * torch.tensor([0.98, 0.98, 1.0]) + torch.tensor([x + 0.01, y + 0.01, -0.5]))
        pb += [b] * 40
    for bb in (0, 1, 2, big_b):
        for x, y, _ in cells:
            rois.append([x + 0.5, y + 0.5, -1.0, 0.3, 0.3, 2.0, 0.2])        # enlarged by 0.5: inside the cell
            rb.append(bb)
    pts = torch.cat(pts + [torch.rand((n_target - 40 * len(cells), 3), generator=g) * 5 + 200.0])
    pb = torch.tensor(pb + [0] * (n_target - 40 * len(cells)), dtype=torch.int32)
    rois, rb = torch.tensor(rois), torch.tensor(rb, dtype=torch.int32)
    assert table_size(pts.shape[0]) - 1 == mask
    dpp_poison(c)
    got = dpp_abi(c, rois, pts, RP_MAX_INBOX, 10 ** 5, rb=rb, pb=pb)
    check_dpp(got, dpp_expect(rois, pts, RP_MAX_INBOX, 10 ** 5, rb=rb, pb=pb), rois, lambda i: pts[i])
    assert torch.equal(rb[got[1]], pb[got[0]])
    pairs = got[1] * pts.shape[0] + got[0]
    assert torch.unique(pairs).numel() == pairs.numel()
    assert got[0].numel() > 0 and {0, 1, big_b} <= set(rb[got[1]].tolist())
    feats = torch.randn((pts.shape[0], 33), generator=g)
    for mode in (0, 1):
        pooled, st, dense = check_pool(c, rois, pts, feats, (2, 2, 2), 16, mode, rb=rb, pb=pb)


# ---- RoIAwarePool3d ------------------------------------------------------------------------------------------------------------------
def _crowd_frame(seed, n_rois=12):
    """a frame, plus a crowded voxel of 40 points (random indices) in RoI 0, with ties, NaN and -inf in its features"""
    pts, rois, _, _ = RO.synth_roi_frame(seed, n_pts=3000, n_rois=n_rois, spread=6.0)
    g = torch.Generator().manual_seed(seed)
    cz = rois[0, 2] + rois[0, 5] / 2
    crowd = torch.tensor([rois[0, 0] + 0.17, rois[0, 1] + 0.13, cz + 0.11]) + (torch.rand((40, 3), generator=g) - 0.5) * 0.006
    pts = torch.cat([pts, crowd])
    perm = torch.randperm(pts.shape[0], generator=g)
    return pts[perm], rois, torch.argsort(perm)[-40:]


def _feats(N, Ch, seed, crowd):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn((N, Ch), generator=g) * 10.0 ** torch.randint(-2, 3, (N, Ch), generator=g).float()
    f[crowd[::3]] = f[crowd[0]].clone()                  # ties
    f[crowd[1::7], 0] = float("nan")
    f[crowd[2::5]] = -float("inf")
    return f


@pytest.mark.parametrize("out_size", [(1, 1, 1), (3, 3, 7), (4, 4, 4), (5, 13, 1), (3, 5, 17), (4, 8, 8), (1, 1, 255)])
@pytest.mark.parametrize("mode", [0, 1])
def test_pool3d_voxels_and_channels(cuda, out_size, mode):
    """nvox around powers of two, C around 32, m = 1 / 2 / 5 / 128 with a crowded voxel keeping its lowest indices"""
    L = _L()
    c = L.ctx(cuda)
    nvox = out_size[0] * out_size[1] * out_size[2]
    assert nvox in (1, 63, 64, 65, 255, 256)
    pts, rois, crowd = _crowd_frame(nvox + mode)
    for j, Ch in enumerate((1, 31, 32, 33, 64, 65, 257)):
        m = (1, 2, 5, 128)[j % 4]
        feats = _feats(pts.shape[0], Ch, j, crowd)
        pooled, st, dense = check_pool(c, rois, pts, feats, out_size, m, mode, grad=Ch <= 65)
        K = int(st[4][1].item())
        if m == 1:
            assert K == 0 and (pooled == 0).all()
        elif m <= 5:
            vox = dense[0].reshape(-1, m)
            full = (vox[:, 0] == m - 1).nonzero()[:, 0]
            assert full.numel() > 0                                            # the crowded voxel is cut to its m - 1 lowest indices
            if nvox == 1:
                assert torch.equal(vox[0, 1:].long(), RA.membership(pts, rois[:1])[0][0].nonzero()[:m - 1, 0])
    rc, P = ra_plan(c, rois, pts, (255, 255, 255), 8)
    assert rc == 0 and P == int(RA.membership(pts, rois)[0].sum())


def test_pool3d_warp_edges(cuda):
    """one voxel per RoI and 200 RoIs: occupied slots 31 | 32 and 63 | 64 with whole empty 32-slot warps between the others"""
    L = _L()
    c = L.ctx(cuda)
    R = 200
    occ = [31, 32, 63, 64, 130, 199]
    k = torch.arange(R).float()
    rois = torch.stack([k * 10.0, torch.zeros_like(k), torch.full_like(k, -1.0), torch.full_like(k, 2.0), torch.full_like(k, 2.0),
                        torch.full_like(k, 2.0), torch.zeros_like(k)], 1)
    g = torch.Generator().manual_seed(3)
    pts = torch.cat([torch.tensor([r * 10.0, 0.0, 0.0]) + (torch.rand((5, 3), generator=g) - 0.5) * 1.5 for r in occ])
    pts = pts[torch.randperm(pts.shape[0], generator=g)]
    for Ch in (1, 31, 32, 33, 65):
        for mode in (0, 1):
            feats = torch.randn((pts.shape[0], Ch), generator=g)
            pooled, st, dense = check_pool(c, rois, pts, feats, (1, 1, 1), 4, mode)
            V = int(st[4][0].item())
            slots = st[0][:V].cpu().tolist()
            assert slots == occ
            warps = {s // 32 for s in slots}
            assert {3, 5} & warps == set() and {0, 1, 2, 4, 6} <= warps
            assert (pooled.reshape(R, -1)[[r for r in range(R) if r not in occ]] == 0).all()


def test_pool3d_clamped_voxel_index(cuda):
    """points on the top face (index oz, clamped to oz - 1), one fp32 step inside the +l/2 face (rounds to ox), below the bottom but
    admitted by the rounded centre (index 0), and NaN z (index 0)"""
    L = _L()
    c = L.ctx(cuda)
    rois = torch.tensor([[0.0, 0.0, -1.0000001, 2.0, 4.0, 1.7, 0.0], [10.0, 0.0, 0.3, 3.0, 3.0, 0.9, math.pi / 2]])
    pts = []
    for r in rois.tolist():
        cx, cy, zb, w, l, h, _ = r
        top = float(np.float32(zb) + np.float32(h))
        pts += [[cx, cy, top], [cx + 0.3, cy - 0.2, top], [cx, cy, zb], [cx, cy, float(np.nextafter(np.float32(zb), np.float32(-9)))]]
        pts += [[cx + float(np.nextafter(np.float32(w / 2), np.float32(0))), cy, zb + h / 2],
                [cx, cy + float(np.nextafter(np.float32(l / 2), np.float32(0))), zb + h / 2], [cx, cy, float("nan")]]
    pts = torch.tensor(pts, dtype=torch.float32)
    ins = RA.membership(pts, rois)[0]
    for out_size in ((4, 4, 4), (3, 5, 7)):
        for mode in (0, 1):
            feats = torch.randn((pts.shape[0], 3), generator=torch.Generator().manual_seed(mode))
            check_pool(c, rois, pts, feats, out_size, 8, mode)
        _, lx, ly = RA.membership(pts, rois)
        zi = RA.voxel_index(rois, lx, ly, pts[:, 2], out_size) % out_size[2]
        raw_z = (pts[None, :, 2] - rois[:, 2:3]) / (rois[:, 5:6] / out_size[2])
        assert ((raw_z >= out_size[2]) & ins).any() and (zi[(raw_z >= out_size[2]) & ins] == out_size[2] - 1).all()
    assert ins[:, -1].any() or ins[:, 6].any()


def test_pool3d_batched_empty_samples(cuda):
    """batch ids with a sample that has no points, one with no RoIs, one with neither"""
    L = _L()
    c = L.ctx(cuda)
    pts, rois, pb, rb = RO.synth_roi_frame(61, n_pts=8000, n_rois=40, spread=8.0, batch_size=4)
    keep_p, keep_r = pb != 1, rb != 2
    pts, pb, rois, rb = pts[keep_p], pb[keep_p], rois[keep_r], rb[keep_r]
    rb = torch.where(rb == 3, torch.full_like(rb, 5), rb)
    pb = torch.where(pb == 3, torch.full_like(pb, 5), pb)
    feats = torch.randn((pts.shape[0], 16), generator=torch.Generator().manual_seed(2))
    for mode in (0, 1):
        pooled, st, dense = check_pool(c, rois, pts, feats, (6, 4, 3), 16, mode, rb=rb, pb=pb)
        assert (pooled[rb == 1] == 0).all() and pooled[rb == 0].abs().sum() > 0


@pytest.mark.parametrize("N", [255, 256, 65535, 65536])
def test_pool3d_backward_pad_key(cuda, N):
    """N = 2^k - 1 | 2^k: the sort's bits_for(N + 1) changes; points 0 and N - 1 are held, most pairs are not kept (m = 2), and one
    point sits in 50 overlapping RoIs"""
    L = _L()
    c = L.ctx(cuda)
    assert bits_for(N + 1) == {255: 8, 256: 9, 65535: 16, 65536: 17}[N]
    g = torch.Generator().manual_seed(N)
    n_in = 240
    pts = torch.rand((N, 3), generator=g) * 50 + 500.0
    inner = torch.cat([torch.tensor([0, 1, N - 1]), 2 + torch.randperm(N - 3, generator=g)[:n_in - 3]])
    pts[inner] = torch.rand((n_in, 3), generator=g) * torch.tensor([2.0, 2.0, 1.0]) - torch.tensor([1.0, 1.0, 0.5])
    pts[0], pts[1], pts[N - 1] = torch.tensor([0.3, -0.2, 0.1]), torch.tensor([0.05, 0.05, 0.0]), torch.tensor([-0.4, 0.35, -0.2])
    base = torch.tensor([0.0, 0.0, -1.0, 2.2, 2.2, 2.0, 0.0])
    rois = base.repeat(50, 1)
    rois[:, 3:5] += torch.arange(50)[:, None] * 0.01
    rois[:, 6] = torch.arange(50) * 0.03
    for m, mode in ((2, 1), (2, 0), (128, 1)):
        feats = torch.randn((N, 3), generator=g)
        pooled, st, dense = check_pool(c, rois, pts, feats, (3, 3, 2), m, mode)
        P, K = st[5], int(st[4][1].item())
        held = dense.reshape(-1, m)
        pts_held = set(held[held[:, 0] > 0][:, 1:].flatten().tolist())
        assert 0 in pts_held and (N - 1 in pts_held or m == 2)
        if m == 2:
            assert K * 4 < P
        if m == 128:
            assert int((held[:, 1:] == 1).sum()) == 50                         # point 1: one voxel in each of the 50 RoIs


def test_pool3d_key_bits(cuda):
    """RoI, voxel and point bits summing to exactly 64 are planned; 65 are refused before any work"""
    L = _L()
    c = L.ctx(cuda)
    out = (255, 255, 255)
    N = 1 << 19
    R = 1 << 21
    assert bits_for(R) + bits_for(255 ** 3) + bits_for(N) == 64 and bits_for(R + 1) + bits_for(255 ** 3) + bits_for(N) == 65
    rois = torch.zeros((R + 1, 7), device="cuda")
    pts = torch.full((N, 3), 900.0, device="cuda")
    rc, P = ra_plan(c, rois[:R], pts, out, 8)
    assert rc == 0 and P == 0
    rc, P = ra_plan(c, rois, pts, out, 8)
    assert rc == ERR_UNSUPPORTED and P == -7
