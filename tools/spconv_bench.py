"""FSD sparse U-Net (SURVEY 8f next-1) on one GPU: SimpleSparseUNet with the configs/fsd/fsd_waymoD1_1x.py backbone shape on a
150k-point synthetic sweep voxelised at 0.2 m (grid 32 x 640 x 640), eval mode.  Reports table building + forward time for the
FFMA path and the wgmma path, per-convolution FLOPs / bytes and the achieved rates.  No oracle import.

    python tools/spconv_bench.py [--reps 10] [--out FILE.json] [--once precision]   (--once: one forward, for ncu)"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sst_b200.flagship import FSD_UNET, fsd_sweep_voxels  # noqa: E402


def sweep_voxels(dev, shuffle=False):
    feats, coors = fsd_sweep_voxels(shuffle=shuffle)
    return feats.to(dev), coors.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--once", default=None)
    ap.add_argument("--shuffle", action="store_true", help="rows in random order instead of the voxel encoder's sorted order")
    a = ap.parse_args()
    from sst_b200 import registry, spconv_modules as SP
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    net = registry.MODELS.build(dict(FSD_UNET)).to(dev).eval()
    feats, coors = sweep_voxels(dev, shuffle=a.shuffle)
    info = dict(voxel_feats=feats, voxel_coors=coors)

    # per-convolution work: record (n_out, pairs, cin, cout) of every launch
    launches = []
    real = SP.indice_conv

    def spy(features, nbr, weight, *args, **kw):
        launches.append((nbr.shape[0], int((nbr >= 0).sum()), weight.shape[1], weight.shape[2], nbr.shape[1]))
        return real(features, nbr, weight, *args, **kw)

    if a.once:
        SP.set_spconv_precision(net, a.once)
        with torch.no_grad():
            net(info)
            torch.cuda.synchronize()
            torch.cuda.cudart().cudaProfilerStart()
            net(info)
            torch.cuda.synchronize()
            torch.cuda.cudart().cudaProfilerStop()
        return
    SP.indice_conv = spy
    with torch.no_grad():
        net(info)
    SP.indice_conv = real
    flops = sum(2 * p * ci * co for _, p, ci, co, _ in launches)
    dense_flops = sum(2 * n * kv * ci * co for n, _, ci, co, kv in launches)
    byts = sum(p * ci * 4 + n * co * 4 + n * kv * 4 + kv * ci * co * 4 for n, p, ci, co, kv in launches)

    def timed(fn, reps):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    res = dict(workload="SimpleSparseUNet configs/fsd shape, 150k-point sweep -> %d voxels, grid 32x640x640, eval" % coors.shape[0],
               row_order="shuffled" if a.shuffle else "sorted (z,y,x)", voxels=int(coors.shape[0]), conv_launches=len(launches), pair_gflop=flops / 1e9, dense_tile_gflop=dense_flops / 1e9,
               algorithmic_mb=byts / 1e6)
    with torch.no_grad():
        for prec in ("fp32", "bf16", "fp32_tc"):
            SP.set_spconv_precision(net, prec)
            ms = timed(lambda: net(info), a.reps)
            res[prec] = dict(ms_forward_incl_tables=ms, tflops_pairs=flops / ms / 1e9)
        # tables alone: one SubM table + one strided pair of tables at the input resolution
        shape = FSD_UNET["sparse_shape"]
        res["table_subm_ms"] = timed(lambda: SP.conv_table(coors, coors, 1, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1]), a.reps)
        oshape = SP.get_conv_output_size(shape, [3, 3, 3], [2, 2, 2], [1, 1, 1], [1, 1, 1])
        res["out_coors_ms"] = timed(lambda: SP.conv_out_coors(coors, 1, shape, oshape, [3, 3, 3], [2, 2, 2], [1, 1, 1]), a.reps)
        # the input-resolution SubM convolution alone (64 -> 64), both paths
        nbr, _ = SP.conv_table(coors, coors, 1, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
        w = torch.randn((27, 64, 64), device=dev) * 0.02
        pairs = int((nbr >= 0).sum())
        for prec in ("fp32", "bf16", "fp32_tc"):
            w16 = SP._pack_h16(w, prec) if prec != "fp32" else None
            ms = timed(lambda: SP.indice_conv(feats, nbr, w, w16, precision=prec), a.reps * 3)
            res[f"subm64_{prec}"] = dict(us=ms * 1e3, pairs=pairs, tflops_pairs=2 * pairs * 64 * 64 / ms / 1e9,
                                         tflops_dense_tile=2 * coors.shape[0] * 27 * 64 * 64 / ms / 1e9,
                                         gbps_gather=(pairs * 256 + coors.shape[0] * (256 + 108)) / ms / 1e6)
    print(json.dumps(res))
    if a.out:
        with open(os.path.join(ROOT, a.out), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
