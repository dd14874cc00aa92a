"""The reference's OWN compiled voxel_layer (oracle/_ref/voxel_layer_ref.so: /root/reference/mmdet3d/ops/voxel/src/*.cpp,*.cu
built unmodified for sm_90a by oracle/build_ref.py) as the checker:

  * CPU (not gpu): pins oracle.dynamic_voxelize to the reference C++ `dynamic_voxelize` (voxelization_cpu.cpp:7-41).
  * GPU: libsstb200 vs the reference CUDA kernels on the same GPU - `dynamic_voxelize_gpu` (voxelization_cuda.cu:332-375)
    and `dynamic_point_to_voxel_forward/backward_gpu` (scatter_points_cuda.cu:183-303); indices bit-exact.

Skipped when the prebuilt extension is absent (it is git-ignored, travels with gpurun, and is rebuilt by
__graft_entry__.build() wherever /root/reference exists)."""
import pytest
import torch

from oracle import build_ref, sst_oracle as O

VS = (0.32, 0.32, 6)
RNG = [-74.88, -74.88, -2, 74.88, 74.88, 4]


@pytest.fixture(scope="module")
def ref():
    try:
        m = build_ref.load_module()
    except Exception as e:  # e.g. a torch ABI mismatch
        pytest.skip(f"oracle/_ref not loadable: {e}")
    if m is None:
        pytest.skip("oracle/_ref/voxel_layer_ref.so not built")
    return m


@pytest.mark.parametrize("voxel_size,rng", [(VS, RNG), ((0.25, 0.25, 0.2), [-80, -80, -2, 80, 80, 4]),
                                             ((0.1, 0.1, 0.15), [-51.2, -51.2, -5, 51.2, 51.2, 3])])
def test_oracle_voxelize_equals_reference_cpp(ref, voxel_size, rng):
    pts = O.synth_frame(11, 40000)
    pts[::7, 0] += 200.0
    pts[::11, 1] -= 300.0
    co = torch.zeros((pts.shape[0], 3), dtype=torch.int32)
    ref.dynamic_voxelize(pts, co, list(voxel_size), list(rng), 3)
    assert torch.equal(co, O.dynamic_voxelize(pts, voxel_size, rng))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 20000, 150000])
def test_voxelize_vs_reference_cuda(cuda, ref, P):
    from sst_b200 import ops
    pts = O.synth_frame(77 + P, P).to(cuda)
    pts[::5, 0] += 300.0
    r = torch.zeros((P, 3), dtype=torch.int32, device=cuda)
    ref.dynamic_voxelize(pts, r, list(VS), list(RNG), 3)
    g = torch.zeros((P, 3), dtype=torch.int32, device=cuda)
    ops.dynamic_voxelize(pts, g, VS, RNG, 3)
    assert torch.equal(r, g)


@pytest.mark.gpu
@pytest.mark.parametrize("reduce", ["max", "mean", "sum"])
@pytest.mark.parametrize("P,C,lo", [(150000, 128, 0), (200000, 3, -1), (5000, 64, -1), (17, 5, 0)])
def test_dynamic_scatter_vs_reference_cuda(cuda, ref, reduce, P, C, lo):
    """Forward + backward against the reference CUDA op (sorted unique + atomics) on identical device tensors."""
    from sst_b200 import ops
    g = torch.Generator().manual_seed(P + C)
    feats = (torch.rand(P, C, generator=g) * 100 - 50).to(cuda)
    if P >= 100000:
        coors = ops.Voxelization(VS, RNG, -1)(O.synth_frame(5, P).to(cuda))
    else:
        coors = torch.randint(lo, 20, (P, 3), generator=g, dtype=torch.int32).to(cuda)
    r_f, r_c, r_m, r_n = ref.dynamic_point_to_voxel_forward(feats, coors, reduce)
    g_f, g_c, g_m, g_n = ops.dynamic_point_to_voxel_forward(feats, coors, reduce)
    assert torch.equal(g_c, r_c) and torch.equal(g_m, r_m) and torch.equal(g_n, r_n)
    if reduce == "max":
        assert torch.equal(g_f, r_f)
    else:  # the reference accumulates with fp32 atomics in arbitrary order
        torch.testing.assert_close(g_f, r_f, rtol=1e-5, atol=2e-3 if reduce == "sum" else 1e-4)
    grad = torch.randn(r_f.shape, generator=g).to(cuda)
    r_g, g_g = torch.zeros_like(feats), torch.zeros_like(feats)
    ref.dynamic_point_to_voxel_backward(r_g, grad, feats, r_f, r_m, r_n, reduce)
    ops.dynamic_point_to_voxel_backward(g_g, grad, feats, r_f, r_m, r_n, reduce)
    torch.testing.assert_close(g_g, r_g, rtol=1e-6, atol=1e-6)


@pytest.mark.gpu
def test_speed_vs_reference_cuda(cuda, ref):
    """SURVEY 8(d): "also time the reference CUDA voxel_layer built for sm_90a - the in-tree GPU kernel to beat for V1/V2".
    Same device tensors, CUDA events, L2 flushed before every call, median of 15.  The gate is deliberately loose (2x); the
    measured ratios are printed (run with -s) and written to gpurun_out/ref_cuda_timing.json when that directory exists."""
    import json
    import os
    from sst_b200 import ops
    P, C = 150000, 128
    pts = O.synth_frame(1000, P).to(cuda)
    coors = ops.Voxelization(VS, RNG, -1)(pts)
    feats = torch.randn(P, C, device=cuda)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=cuda)

    def timed(fn, iters=15):
        ts = []
        for i in range(iters + 2):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            if i >= 2:
                ts.append(a.elapsed_time(b) * 1e3)
        return sorted(ts)[len(ts) // 2]

    out = {}
    rc = torch.zeros((P, 3), dtype=torch.int32, device=cuda)
    gc = torch.zeros((P, 3), dtype=torch.int32, device=cuda)
    out["dynamic_voxelize"] = dict(reference_us=timed(lambda: ref.dynamic_voxelize(pts, rc, list(VS), list(RNG), 3)),
                                   ours_us=timed(lambda: ops.dynamic_voxelize(pts, gc, VS, RNG, 3)))
    for red in ("max", "mean"):
        ds = ops.DynamicScatter(VS, RNG, red == "mean")
        out[f"dynamic_scatter_{red}_C{C}"] = dict(
            reference_us=timed(lambda: ref.dynamic_point_to_voxel_forward(feats, coors, red)),
            ours_us=timed(lambda: ds(feats, coors)))
    for k, v in out.items():
        v["speedup"] = v["reference_us"] / v["ours_us"]
        print(f"{k}: reference CUDA {v['reference_us']:.1f} us, libsstb200 {v['ours_us']:.1f} us, x{v['speedup']:.1f}")
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if os.path.isdir(d):
        json.dump(out, open(os.path.join(d, "ref_cuda_timing.json"), "w"), indent=1)
    assert out["dynamic_scatter_max_C128"]["speedup"] > 2.0 and out["dynamic_scatter_mean_C128"]["speedup"] > 2.0


HV_CASES = [  # (P, F, voxel_size, range, max_points, max_voxels)
    (20000, 4, (0.32, 0.32, 6), [-74.88, -74.88, -2, 74.88, 74.88, 4], 32, 20000),
    (20000, 4, (0.32, 0.32, 6), [-74.88, -74.88, -2, 74.88, 74.88, 4], 5, 300),       # both caps bite
    (30000, 5, (0.5, 0.5, 0.25), [-40, -40, -3, 40, 40, 1], 10, 16000),               # 3-D grid
    (7, 3, (1.0, 1.0, 1.0), [0, 0, 0, 4, 4, 4], 2, 3),
]


def _hv_points(P, F):
    pts = O.synth_frame(300 + P, P, extra_dims=F - 3)
    pts[::13, 0] += 500.0  # out of range -> clamped by this fork's voxeliser
    return pts


@pytest.mark.parametrize("P,F,vs,rng,mp,mv", HV_CASES)
def test_oracle_hard_voxelize_equals_reference_cpp(ref, P, F, vs, rng, mp, mv):
    """Pins oracle.hard_voxelize to the reference's own `hard_voxelize_cpu` (voxelization_cpu.cpp:43-142)."""
    pts = _hv_points(P, F)
    voxels = torch.zeros((mv, mp, F))
    coors = torch.zeros((mv, 3), dtype=torch.int32)
    npts = torch.zeros((mv,), dtype=torch.int32)
    n = ref.hard_voxelize(pts, voxels, coors, npts, list(vs), list(rng), mp, mv, 3)
    ov, oc, on = O.hard_voxelize(pts, vs, rng, mp, mv)
    assert n == ov.shape[0]
    assert torch.equal(oc, coors[:n]) and torch.equal(on, npts[:n]) and torch.equal(ov, voxels[:n])


@pytest.mark.gpu
@pytest.mark.parametrize("P,F,vs,rng,mp,mv", HV_CASES + [(150000, 4, (0.32, 0.32, 6), [-74.88, -74.88, -2, 74.88, 74.88, 4], 32, 32000)])
def test_hard_voxelize_vs_reference(cuda, ref, P, F, vs, rng, mp, mv):
    """libsstb200 `Voxelization(max_num_points > 0)` against the reference CPU implementation (bit-exact: pure data movement)."""
    from sst_b200 import ops
    pts = _hv_points(P, F)
    voxels = torch.zeros((mv, mp, F))
    coors = torch.zeros((mv, 3), dtype=torch.int32)
    npts = torch.zeros((mv,), dtype=torch.int32)
    n = ref.hard_voxelize(pts, voxels, coors, npts, list(vs), list(rng), mp, mv, 3)
    layer = ops.Voxelization(vs, rng, mp, mv).eval()
    gv, gc, gn = layer(pts.to(cuda))
    assert gv.shape[0] == n
    assert torch.equal(gc.cpu(), coors[:n]) and torch.equal(gn.cpu(), npts[:n]) and torch.equal(gv.cpu(), voxels[:n])
