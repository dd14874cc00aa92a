"""sstb200_hard_voxelize on a fresh context at point counts whose workspace lands just below an arena capacity.

The arena starts at 16 MiB and doubles to the first power of two that holds a call's workspace, so a point count whose workspace
ends just below 32, 64 or 128 MiB runs in an arena with almost no headroom.  Each count gets its own context straight from
sstb200_create (so the arena is sized by this call alone) and is freed with sstb200_destroy.  The points sit at the centres of a
64 x 64 voxel grid in first-occurrence order, so the voxels, their coordinates and their point counts are known exactly."""
import ctypes as C

import numpy as np
import pytest
import torch

from sst_b200 import _lib as L

pytestmark = pytest.mark.gpu

NX = NY = 64
MAX_POINTS = 5
F = 4
MIB = 1 << 20


def al256(b):
    return (b + 255) // 256 * 256


def workspace_estimate(P):
    """hard_voxelize's arena bytes at P points, with cub's radix-sort scratch taken as two P-element key / value buffers."""
    scan = lambda n: al256(256 + ((n + 1 + 2047) // 2048 + 1) * 8)
    T = NX * NY
    nwords = (T + 31) // 32
    pwords = (P + 31) // 32
    key_index = al256(P * 8) + al256(nwords * 4) + scan(nwords) + al256((nwords + 1) * 4)
    return (key_index + al256(P * 12) + 8 * al256(P * 4 + 8) + al256(pwords * 4) + scan(pwords) + scan(P) + al256((pwords + 2) * 4) +
            al256(8 * P + 16))


def counts_below(cap):
    """point counts whose workspace ends from about 3 MiB below `cap` up to just past it"""
    lo, hi = 1, 1 << 26
    while lo < hi:  # largest P with estimate <= cap
        mid = (lo + hi + 1) // 2
        if workspace_estimate(mid) <= cap:
            lo = mid
        else:
            hi = mid - 1
    per_point = (workspace_estimate(lo) - workspace_estimate(lo - 10000)) / 10000
    step = int(256 * 1024 / per_point)
    return [lo - k * step for k in range(12, -2, -1)]


SWEEP = [P for cap in (32 * MIB, 64 * MIB, 128 * MIB) for P in counts_below(cap)]


@pytest.mark.parametrize("P", SWEEP)
def test_hard_voxelize_fresh_context(P):
    dev = torch.device("cuda:0")
    cell = torch.arange(P, dtype=torch.int64) % (NX * NY)
    x, y = (cell % NX).float() + 0.5, (cell // NX).float() + 0.5
    pts = torch.stack([x, y, torch.full_like(x, 0.5), torch.arange(P, dtype=torch.float32)], 1).to(dev)
    V = NX * NY
    voxels = torch.zeros((V, MAX_POINTS, F), dtype=torch.float32, device=dev)
    coors = torch.zeros((V, 3), dtype=torch.int32, device=dev)
    npv = torch.zeros((V,), dtype=torch.int32, device=dev)
    num_dev = torch.empty((1,), dtype=torch.int32, device=dev)
    num = C.c_int32(-1)
    lib = L.lib()
    torch.cuda.synchronize()
    c = lib.sstb200_create(0)
    assert c
    try:
        rc = lib.sstb200_hard_voxelize(c, pts.data_ptr(), P, F, L.arr(C.c_float, [1.0, 1.0, 1.0]),
                                       L.arr(C.c_float, [0.0, 0.0, 0.0, float(NX), float(NY), 1.0]), MAX_POINTS, V, voxels.data_ptr(),
                                       coors.data_ptr(), npv.data_ptr(), num_dev.data_ptr(), C.byref(num))
        msg = lib.sstb200_last_error(c)
        assert rc == 0, f"P = {P}: {msg.decode() if msg else '?'}"
    finally:
        lib.sstb200_destroy(c)
    assert num.value == V and int(num_dev.item()) == V
    v = np.arange(V)
    expect = np.stack([np.zeros(V, np.int32), v // NX, v % NX], 1)
    assert np.array_equal(coors.cpu().numpy(), expect)
    assert torch.equal(npv.cpu(), torch.full((V,), MAX_POINTS, dtype=torch.int32))
    # each voxel keeps its first MAX_POINTS points in input order: point ids v, v + V, v + 2V, ...
    ids = voxels[:, :, 3].cpu().numpy()
    assert np.array_equal(ids, v[:, None] + V * np.arange(MAX_POINTS)[None, :])
