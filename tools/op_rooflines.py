"""Per-op latency + roofline table for every SURVEY.md 8(a) row, through the public Python ops / modules (the calls a
reference user makes), on config-2 / config-3 shapes.  CUDA events on the current stream, L2 flushed before every call,
median of `--iters`.  Ops that return data-dependent shapes read one int32 back (like the reference) - that sync is inside
the timing, so these are API latencies, not kernel sums (kernel sums: torch.profiler launch lists).  The reference's own
CUDA voxel_layer is timed on the same tensors by tests/test_ref_voxel_layer.py::test_speed_vs_reference_cuda.

    python tools/op_rooflines.py [--iters 20] [--out gpurun_out/op_rooflines.json]
    ncu ... python tools/op_rooflines.py --once        # one call per op, separated by marker kernels (torch.arange)
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sst_b200 import flagship as fl, ops  # noqa: E402
from sst_b200.sir_modules import SIR  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--once", action="store_true")
ap.add_argument("--out", default=None)
args = ap.parse_args()
dev = torch.device("cuda:0")
P, C = 150000, 128
pk = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) \
    if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else \
    {"hbm_gbs": 6650.0, "bf16_tflops_sustained": 1400.0}
flush_buf = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def timed(fn, iters):
    ts = []
    for i in range(iters + 2):
        flush_buf.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= 2:
            ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


rows = []


def op(name, ref, fn, bytes_=None, flops=None, note=""):
    if args.once:
        fn()
        torch.cuda.synchronize()
        torch.arange(7, device=dev)  # marker kernel between ops
        fn()
        torch.cuda.synchronize()
        torch.arange(7, device=dev)
        print("once:", name)
        return
    us = timed(fn, args.iters)
    r = {"op": name, "reference": ref, "us": round(us, 2), "note": note}
    if bytes_:
        r.update(algorithmic_bytes=int(bytes_), gbs=round(bytes_ / us / 1e3, 1),
                 hbm_frac=round(bytes_ / us / 1e3 / pk["hbm_gbs"], 4))
    if flops:
        r.update(flops=int(flops), tflops=round(flops / us / 1e6, 2),
                 tensor_frac=round(flops / us / 1e6 / pk["bf16_tflops_sustained"], 4))
    rows.append(r)
    print(json.dumps(r), flush=True)


with torch.no_grad():
    pts = fl.synth_frame(1000, P).to(dev)
    vox = ops.Voxelization(fl.VOXEL_SIZE, fl.PC_RANGE, -1).to(dev)
    op("V1 Voxelization(dynamic)", "ops/voxel/voxelize.py:102-113", lambda: vox(pts), bytes_=P * (3 * 4 + 3 * 4))
    coors3 = vox(pts)
    hvox = ops.Voxelization(fl.VOXEL_SIZE, fl.PC_RANGE, 32, 32000).to(dev).eval()
    op("V1' Voxelization(hard, max_points=32, max_voxels=32000)", "ops/voxel/voxelize.py:45-57 -> src/voxelization_cuda.cu:188-330",
       lambda: hvox(pts), bytes_=P * 12 + 32000 * 32 * 12, note="bytes = read points + the zero-filled [max_voxels, max_points, F] output")
    feats = torch.randn(P, C, device=dev)
    M = ops.dynamic_point_to_voxel_forward(feats, coors3, "max")[0].shape[0]
    v2_bytes = P * (4 * C + 12) + M * (4 * C + 12) + 4 * P + 4 * M
    for red in ("max", "mean"):
        ds = ops.DynamicScatter(fl.VOXEL_SIZE, fl.PC_RANGE, red == "mean")
        op(f"V2 DynamicScatter({red}, C={C})", "ops/voxel/scatter_points.py:52-110 -> src/scatter_points_cuda.cu:183-234",
           lambda ds=ds: ds(feats, coors3), bytes_=v2_bytes, note=f"M={M}")
    red_f, out_c, cmap, cnt = ops.dynamic_point_to_voxel_forward(feats, coors3, "max")
    gout = torch.randn_like(red_f)
    gin = torch.zeros_like(feats)
    op("V3 dynamic_point_to_voxel_backward(max)", "ops/voxel/src/scatter_points_cuda.cu:236-303",
       lambda: ops.dynamic_point_to_voxel_backward(gin, gout, feats, red_f, cmap, cnt, "max"),
       bytes_=P * 4 * C * 2 + M * 4 * C * 2 + 4 * P, note="reads feats+reduced+grad_reduced, writes grad_feats")
    coors4 = torch.cat([torch.zeros(P, 1, dtype=torch.int32, device=dev), coors3], 1)
    c64 = coors4.long()
    op("V5 scatter_v2(max, C=128, int64 coors)", "ops/sst/sst_ops.py:151-182", lambda: ops.scatter_v2(feats, c64, "max"),
       bytes_=P * (4 * C + 32) + M * (4 * C + 32) + 8 * P)
    op("V5' unique_rows (torch.unique dim=0 + inverse)", "ops/sst/sst_ops.py:158", lambda: ops.unique_rows(c64),
       bytes_=P * 32 + M * 32 + 8 * P)
    vfe, il, bb = fl.build_sst(fl.sst_cfg())
    vfe, bb = vfe.to(dev), bb.to(dev)
    for prec in ("fp32", "bf16"):
        vfe.precision = prec
        op(f"V4 DynamicVFE(3->[64,128], {prec})", "models/voxel_encoders/voxel_encoder.py:229-298", lambda: vfe(pts, coors4),
           bytes_=P * 28 + M * (4 * C + 16), flops=2 * P * (9 * 64 + 128 * 128))
    vf, vc = vfe(pts, coors4)
    vc = vc.long()
    op("B7 SSTInputLayerV2.forward (B1-B5, both shifts)", "models/middle_encoders/sst_input_layer_v2.py:79-126",
       lambda: il(vf, vc, 1), bytes_=M * (4 * 8 + 6 * 8), note="latency-bound by definition (SURVEY 8d)")
    info = il(vf, vc, 1)
    win = info["batch_win_inds_shift0"]
    op("B2 get_inner_win_inds", "ops/sst/sst_ops.py:244-264", lambda: ops.get_inner_win_inds(win), bytes_=M * 16)
    f2w = info["flat2win_inds_shift0"]
    op("B6 flat2window_v2", "ops/sst/sst_ops.py:141-149", lambda: ops.flat2window_v2(vf, f2w), bytes_=2 * M * C * 4,
       note="compat layout only; the SRA kernels never materialise it")
    w3 = ops.flat2window_v2(vf, f2w)
    op("B6 window2flat_v2", "ops/sst/sst_ops.py:67-132", lambda: ops.window2flat_v2(w3, f2w), bytes_=2 * M * C * 4)
    sn2 = float(sum((torch.bincount(info[f"batch_win_inds_shift{s}"]).double() ** 2).sum().item() for s in (0, 1)) / 2)
    lflops = M * (8 * C * C + 4 * C * 256) + 4 * C * sn2
    for prec in ("fp32", "bf16"):
        bb.precision = prec
        op(f"A4 SSTv2.forward (12 encoder layers, {prec})", "models/backbones/sst_v2.py:115-154", lambda: bb(info),
           flops=12 * lflops, bytes_=12 * 2 * M * C * 4)
    bbv = fl.build_sst(fl.sst_cfg())[2].to(dev)
    bbv.output_shape = [468, 468]
    xs = bb(info)[0]["voxel_feats"]
    op("A4' SSTv2.recover_bev (B=1, C=128, 468x468)", "models/backbones/sst_v2.py:161-196", lambda: bbv.recover_bev(xs, vc, 1),
       bytes_=128 * 468 * 468 * 4 + M * 128 * 4, note="write-once canvas (zeros included) + one read of the rows")
    # config 3: SIR
    N, G = 150000, 256
    g = torch.Generator().manual_seed(3)
    sp = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1).to(dev)
    sf = torch.randn(N, 79, generator=g).to(dev)
    gid = torch.randint(0, G, (N,), generator=g)
    sc = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1).to(dev)
    fcl = (torch.randn(N, 3, generator=g) * 2).to(dev)
    torch.manual_seed(0)
    sir = SIR(num_blocks=3, in_channels=[84, 133, 133], feat_channels=[[128, 128]] * 3, rel_mlp_hidden_dims=[[16, 32]] * 3,
              norm_cfg=dict(type="LN", eps=1e-3), mode="max", xyz_normalizer=[20, 20, 4], act="gelu",
              unique_once=True).eval().to(dev)
    sflops = 0
    for cin in (84, 133, 133):
        sflops += 2 * N * (3 * 16 + 16 * 32 + 32 * cin + cin * 128 + 256 * 128)
    for prec in ("fp32", "bf16"):
        sir.precision = prec
        op(f"S2 SIR.forward (config 3: 150k pts, 256 groups, 3 blocks, {prec})", "models/backbones/sir.py:67-87",
           lambda: sir(sp, sf, sc, fcl), flops=sflops, bytes_=N * (84 + 128) * 4 + 3 * G * 256 * 4,
           note="bytes = read [points|feats] once + write point feats once; intermediates counted as on-chip")

if args.out and not args.once:
    json.dump({"peaks": pk, "rows": rows}, open(args.out, "w"), indent=1)
